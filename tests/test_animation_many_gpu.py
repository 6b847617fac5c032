"""lb200_animation_update_many (AnimationSystem.updateMany): every system of a frame posed in one launch, bit for bit what per-system
updates give.

Every system is built twice from the same inputs: one twin goes through updateMany, the other through update, and every output the
frame asked for (dual quaternions, matrices, absolute poses, advanced times) must be byte-equal.  The first frame of the shape mix is
also held to the oracle directly.  Then the launch shape (one G per call, the 4-lane fallback, what get_launch reports), lists longer
than one launch, the refusals, the consumers of the poses (skin, bone attachments, compute_relative, propagate_attached) and the engine
binding over several real Models (oracle/_ref, skipped when it is not built).
"""
import ctypes as C
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from bitexact import assert_bits_equal
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

DQ, MTX, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_MATRIX, lb.PALETTE_POSE
ALL = DQ | MTX | POSE
CAP = 64  # systems per launch (POSE_MANY_CAP in csrc/animation.cu)
ERR_INVALID = lb._lib.ERR_INVALID


def _random_tree(n, seed):
    rng = np.random.default_rng(seed)
    return [-1] + [int(rng.integers(0, i)) for i in range(1, n)]


def _five_root_forest():
    rng = np.random.default_rng(11)
    parents = [-1] * 5 + [r for r in range(5) for _ in range(8)]
    for i in range(len(parents), 70):
        parents.append(int(rng.integers(5, i)))
    return parents


SHAPES = {
    "1": [-1],
    "3": [-1, 0, 1],
    "all_roots": [-1] * 7,
    "five_roots": _five_root_forest(),
    "star196": [-1] + [0] * 195,
    "chain192": [-1] + list(range(191)),
    "chain196": [-1] + list(range(195)),
    "random150": _random_tree(150, 5),
    "c4_64": None,
}


def _skeleton(name):
    parents = SHAPES[name]
    return scenes.skeleton(64, seed=4) if parents is None else scenes.skeleton(seed=len(parents), parents=parents)


def _clips(sk, seed=21):
    return [scenes.clip(sk, frames=13, fps=30.0, seed=seed, const_fraction=0.3),
            scenes.clip(sk, frames=40, fps=24.0, seed=seed + 1, pos_bits=(11, 14, 16), rot_bits=(12, 15, 16), const_fraction=0.3)]


def _times(n, clips, seed):
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    lengths = np.array([c.length_ticks for c in clips], np.int64)[ci]
    tt = (rng.random(n) * lengths).astype(np.int64)
    for k, f in enumerate([lambda L: 0, lambda L: L - 1, lambda L: L, lambda L: L + 4000][:n]):
        tt[k] = f(lengths[k])
    return ci, tt.astype(np.uint32)


class Twin:
    """One set of inputs, two systems: `many` is updated through updateMany, `one` through update."""

    def __init__(self, ctx, sk, clips, n, seed, lanes=0, layers=0, mesh=None, max_instances=None):
        self.sk, self.clips, self.n = sk, clips, n
        self.ci, self.tt = _times(n, clips, seed)
        self.many = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=max(1, max_instances or n))
        self.one = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=max(1, max_instances or n))
        for s in (self.many, self.one):
            s.setLaunch(pose_lanes=lanes)
            if n:
                s.setInstances(self.ci, self.tt)
        self.layers = layers
        if layers and n:
            rng = np.random.default_rng(seed + 1)
            lci = rng.integers(0, len(clips), (n, layers)).astype(np.uint32)
            ltt = (rng.random((n, layers)) * 2000).astype(np.uint32)
            lw = rng.random((n, layers)).astype(np.float32)
            lw[:, -1] = np.array([0.5, 1.0, 0.99995, 0.9999], np.float32)[np.arange(n) % 4]
            for s in (self.many, self.one):
                s.setLayers(lci, ltt, lw)

    def outputs(self, s, flags):
        if not self.n:
            return {}
        out = {"times": s.getTimes()}
        if flags & DQ:
            out["dq"] = s.getDualQuats()
        if flags & MTX:
            out["mtx"] = s.getMatrices()
        if flags & POSE:
            out["pos"], out["rot"] = s.getPose()
        return out

    def check(self, flags, what):
        a, b = self.outputs(self.many, flags), self.outputs(self.one, flags)
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), f"{what}: {k} of updateMany differs from update"

    def close(self):
        self.many.close()
        self.one.close()


def _frame(twins, dt, flags):
    lb.AnimationSystem.updateMany([t.many for t in twins], dt, flags)
    for t in twins:
        t.one.update(dt, flags)


MIX = ["1", "3", "all_roots", "five_roots", "star196", "chain192", "chain196", "random150", "c4_64"]


def _mix(ctx, lanes, shapes, per_block, big=3000, layered=True):
    counts = [0, 1, per_block - 1, per_block, per_block + 1]
    twins = []
    for k, name in enumerate(shapes):
        sk = _skeleton(name)
        n = big if name == "c4_64" else counts[k % len(counts)]
        layers = (0, 3, 0, 16)[k % 4] if layered else 0
        twins.append(Twin(ctx, sk, _clips(sk, seed=21 + k), n, seed=100 + k, lanes=lanes, layers=layers))
    return twins


def test_shape_mix_against_the_oracle_and_per_system_updates(ctx, oracle):
    twins = _mix(ctx, 0, MIX, 16, layered=False)
    _frame(twins, 1.0 / 60.0, ALL)
    for t in twins:
        t.check(ALL, f"{t.sk.bone_count} bones, {t.n} instances")
        if not t.n:
            continue
        exp = oracle.animate_instances(t.sk, t.clips, t.ci, t.tt)
        pos, rot = t.many.getPose()
        assert_bits_equal(pos, exp["pos"], f"{t.sk.bone_count} bones: pose.pos against the oracle")
        assert_bits_equal(rot, exp["rot"], f"{t.sk.bone_count} bones: pose.rot against the oracle")
        assert_bits_equal(t.many.getDualQuats(), exp["dq"], f"{t.sk.bone_count} bones: dual quats against the oracle")
        assert_bits_equal(t.many.getMatrices(), exp["mtx"], f"{t.sk.bone_count} bones: matrices against the oracle")
        want = np.array([oracle.time_advance(x, 1.0 / 60.0, t.clips[c].fps, t.clips[c].frame_count) for c, x in zip(t.ci, t.tt)], np.uint32)
        assert np.array_equal(t.many.getTimes(), want), f"{t.sk.bone_count} bones: advanced times against the oracle"
    for t in twins:
        assert t.many.lastLaunch()[0] == (8 if t.n else 0)
        t.close()


@pytest.mark.parametrize("lanes", [4, 8, 16, 32])
def test_every_lane_count_palette_and_step(ctx, lanes):
    """G set on every system: that G runs (no skeleton above 192 bones here), over frames with dt > 0, < 0 and 0 and palette flags that
    grow: the second frame's matrices and the third frame's poses are allocated by updateMany itself."""
    shapes = [s for s in MIX if s not in ("star196", "chain196")]
    twins = _mix(ctx, lanes, shapes, 128 // lanes)
    for k, (dt, flags) in enumerate([(1.0 / 30.0, DQ), (-0.3, MTX), (0.0, POSE), (0.75, ALL), (-1.0 / 60.0, DQ | POSE)]):
        _frame(twins, dt, flags)
        for t in twins:
            t.check(flags, f"lanes {lanes}, frame {k}, {t.sk.bone_count} bones, {t.n} instances, {t.layers} layers")
            assert t.many.lastLaunch()[0] == (lanes if t.n else 0)
    for t in twins:
        t.close()


def test_four_lanes_fall_back_with_a_large_skeleton(ctx):
    twins = _mix(ctx, 4, ["3", "star196", "c4_64", "five_roots"], 32, big=500)
    for k, dt in enumerate((0.1, -0.2)):
        _frame(twins, dt, ALL)
        for t in twins:
            t.check(ALL, f"4-lane fallback, frame {k}, {t.sk.bone_count} bones")
            if t.n:
                assert t.many.lastLaunch()[0] == 8
    for t in twins:
        t.close()


def test_disagreeing_settings_run_eight_lanes(ctx):
    sk = _skeleton("five_roots")
    clips = _clips(sk)
    twins = [Twin(ctx, sk, clips, n, seed=n, lanes=lanes) for n, lanes in ((40, 16), (41, 32), (7, 0), (0, 4))]
    _frame(twins, 0.2, ALL)
    for t in twins:
        t.check(ALL, f"mixed lanes, {t.n} instances")
    assert [t.many.lastLaunch()[0] for t in twins] == [8, 8, 8, 0]
    assert [t.one.lastLaunch()[0] for t in twins] == [16, 32, 8, 0]
    for t in twins:
        t.close()


@pytest.mark.parametrize("n_systems", [CAP + 1, 300])
def test_long_lists_split_into_launches(ctx, n_systems):
    sks = [_skeleton(name) for name in ("3", "five_roots", "c4_64")]
    clips = [_clips(sk) for sk in sks]
    twins = [Twin(ctx, sks[k % 3], clips[k % 3], 1 + (k * 7) % 40, seed=k, layers=(k % 5 == 0) * 2) for k in range(n_systems)]
    for k, dt in enumerate((1.0 / 60.0, -0.1, 0.3)):
        before = ctx.launches
        lb.AnimationSystem.updateMany([t.many for t in twins], dt, ALL)
        assert ctx.launches - before == -(-n_systems // CAP)
        for t in twins:
            t.one.update(dt, ALL)
        for i, t in enumerate(twins):
            t.check(ALL, f"{n_systems} systems, frame {k}, system {i}")
    for t in twins:
        t.close()


def test_refusals_change_nothing(ctx):
    sk = _skeleton("c4_64")
    clips = _clips(sk)
    twins = [Twin(ctx, sk, clips, n, seed=n) for n in (5, 33)]
    _frame(twins, 0.1, ALL)
    systems = [t.many for t in twins]
    snap = [t.outputs(t.many, ALL) for t in twins]
    L = lb._lib.lib()

    def unchanged(what):
        for t, s in zip(twins, snap):
            now = t.outputs(t.many, ALL)
            for k in s:
                assert now[k].tobytes() == s[k].tobytes(), f"{what} changed {k}"

    before = ctx.launches
    lb.AnimationSystem.updateMany([], 0.1, ALL)
    assert L.lb200_animation_update_many(None, C.c_uint32(0), C.c_float(0.1), C.c_uint32(ALL)) == 0
    assert ctx.launches == before
    unchanged("n = 0")
    assert L.lb200_animation_update_many(None, C.c_uint32(2), C.c_float(0.1), C.c_uint32(ALL)) == ERR_INVALID
    unchanged("a NULL list")
    ctx2 = lb.Context(0)
    try:
        foreign = lb.AnimationSystem(ctx2, sk, clips, None, max_instances=4)
        foreign.setInstances(*_times(4, clips, 1))
        for bad, what in (([systems[0], None, systems[1]], "a NULL entry"), ([systems[0], systems[1], systems[0]], "a duplicate"),
                          ([systems[0], foreign, systems[1]], "another context's system")):
            with pytest.raises(lb.LumixB200Error) as e:
                lb.AnimationSystem.updateMany(bad, 0.1, ALL)
            assert e.value.code == ERR_INVALID
            unchanged(what)
        assert ctx.launches == before
        assert foreign.getTimes().tobytes() == _times(4, clips, 1)[1].tobytes()
        foreign.close()
    finally:
        ctx2.close()
    for t in twins:
        t.close()


def test_consumers_after_a_batched_update(ctx):
    """skin, bone_attachments_device, compute_relative and propagate_attached read what updateMany wrote as they read update's."""
    from lumixengine_b200.hierarchy import TRANSFORM_DTYPE
    specs = [("c4_64", 37), ("five_roots", 19), ("chain192", 9)]
    twins = []
    for k, (name, n) in enumerate(specs):
        sk = _skeleton(name)
        twins.append(Twin(ctx, sk, _clips(sk, seed=40 + k), n, seed=k, mesh=scenes.mesh(sk, 300, seed=k)))
    _frame(twins, 0.25, ALL)
    for t in twins:
        t.check(ALL, "consumers")
        t.many.skin()
        t.one.skin()
        assert t.many.getSkinned().tobytes() == t.one.getSkinned().tobytes(), "skin after updateMany"
        t.many.computeRelative()
        t.one.computeRelative()
        a, b = t.many.getRelativePose(), t.one.getRelativePose()
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), "compute_relative after updateMany"
    rng = np.random.default_rng(3)
    m = 64
    for t in twins:
        inst = rng.integers(0, t.n, m).astype(np.uint32)
        bone = rng.integers(0, t.sk.bone_count, m).astype(np.uint32)
        rel = np.concatenate([rng.normal(size=(m, 3)), scenes.random_unit_quats(rng, m)], axis=1).astype(np.float32)
        par = np.zeros(m, TRANSFORM_DTYPE)
        par["pos"] = rng.normal(size=(m, 3)) * 100
        par["rot"] = scenes.random_unit_quats(rng, m)
        par["scale"] = 1.0
        sc = (0.5 + rng.random((m, 3))).astype(np.float32)
        dev = [ctx.to_device(x) for x in (inst, bone, rel, par, sc)]
        outs = []
        for s in (t.many, t.one):
            d_out = ctx.to_device(np.zeros(m, TRANSFORM_DTYPE))
            s.boneAttachmentsDevice(m, *dev, d_out)
            outs.append(ctx.copy_to_host(d_out, m * TRANSFORM_DTYPE.itemsize, np.uint8))
            ctx.free_device(d_out)
        for p in dev:
            ctx.free_device(p)
        assert outs[0].tobytes() == outs[1].tobytes(), "bone_attachments_device after updateMany"
    # propagate_attached over the same systems: two identical hierarchies, one reading the batched twins, one the per-system twins
    parents, locals_, roots = scenes.hierarchy_forest(3000, 5, 4, seed=9)
    root_nodes = np.nonzero(np.asarray(parents) < 0)[0]
    k = min(24, len(root_nodes) // 2)
    attached, parent = root_nodes[k:2 * k], root_nodes[:k]
    slot = (np.arange(k) % len(twins)).astype(np.uint32)
    inst = np.array([rng.integers(0, twins[s].n) for s in slot], np.uint32)
    bone = np.array([rng.integers(0, twins[s].sk.bone_count) for s in slot], np.uint32)
    rel = np.concatenate([rng.normal(size=(k, 3)), scenes.random_unit_quats(rng, k)], axis=1).astype(np.float32)
    got = []
    for side in ("many", "one"):
        h = lb.Hierarchy(ctx, parents)
        h.setLocalTransforms(locals_)
        h.setRootTransforms(roots)
        h.propagate()
        h.setAttachments(attached, parent, slot, inst, bone, rel)
        ml = h.propagateAttached([getattr(t, side) for t in twins])
        got.append((h.getTransforms(), ml.count))
        h.close()
    assert got[0][1] == got[1][1] > 0
    for f in ("pos", "rot", "scale"):
        assert got[0][0][f].tobytes() == got[1][0][f].tobytes(), f"propagate_attached after updateMany: {f}"
    for t in twins:
        t.close()


SHIM = po.ANIMATION_SHIM_SO


def test_binding_over_several_models(oracle):
    """host/animation_b200.inl over the animables of three real Lumix::Models of 48, 17 and 130 bones (one group each, all posed by one
    lb200_animation_update_many) against the reference's updateAnimable body per animable, bit for bit."""
    if not os.path.exists(SHIM):
        pytest.skip("oracle/_ref/libanimation_shim_b200.so not built (needs /root/reference at build time)")
    from lumixengine_b200 import _lib
    L = C.CDLL(SHIM)
    os.environ["LB200_ENGINE_SHIM_LOADED"] = "1"  # tests/conftest.py leaves with os._exit once the shim is loaded
    sks = [scenes.skeleton(48, seed=1), scenes.skeleton(17, seed=2), scenes.skeleton(seed=130, parents=_random_tree(130, 7))]
    clips = [[scenes.clip(sk, frames=30 + 5 * j, seed=10 * m + j) for j in range(1 + m)] for m, sk in enumerate(sks)]
    n = 500
    rng = np.random.default_rng(8)
    model_of = rng.integers(0, len(sks), n).astype(np.uint32)
    ci = np.array([rng.integers(0, len(clips[m])) for m in model_of], np.uint32)
    tt = np.array([rng.integers(0, clips[m][c].length_ticks) for m, c in zip(model_of, ci)], np.uint32)
    sk_arr = (_lib.Skeleton * len(sks))(*[sk.as_struct(_lib.Skeleton) for sk in sks])
    flat = [c for cs in clips for c in cs]
    clip_arr = (_lib.Clip * len(flat))(*[c.as_struct(_lib.Clip) for c in flat])
    clip_start = np.cumsum([0] + [len(cs) for cs in clips]).astype(np.uint32)
    bones = sum(sks[m].bone_count for m in model_of)
    out = {k: np.zeros(bones * w, np.float32) for k, w in (("pos_ref", 3), ("rot_ref", 4), ("pos_b", 3), ("rot_b", 4))}
    time_ref, time_b, info = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(4, np.uint32)
    L.ashim_run_models.restype = C.c_int
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for dt, rounds in ((1.0 / 30.0, 3), (-0.05, 2)):
        rc = L.ashim_run_models(sk_arr, C.c_uint32(len(sks)), clip_arr, p(clip_start), p(model_of), p(ci), p(tt), C.c_uint32(n), C.c_float(dt),
                                C.c_uint32(rounds), p(out["pos_ref"]), p(out["rot_ref"]), p(time_ref), p(out["pos_b"]), p(out["rot_b"]), p(time_b), p(info))
        assert rc == 0 and info[2] == 0
        assert info[0] == info[1] == n * rounds and info[3] == n
        assert np.array_equal(time_ref, time_b) and not np.array_equal(time_ref, tt)
        assert out["pos_ref"].tobytes() == out["pos_b"].tobytes(), "AnimablesB200 over several models delivered other bone positions than updateAnimable"
        assert out["rot_ref"].tobytes() == out["rot_b"].tobytes(), "AnimablesB200 over several models delivered other bone rotations than updateAnimable"
        assert np.abs(out["pos_ref"]).max() > 0.1
