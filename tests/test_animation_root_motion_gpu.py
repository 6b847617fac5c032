"""lb200_animation_set_root_motion (AnimationSystem.setRootMotion): clips whose root-motion tracks Animation::setRootMotionBone replaced,
posed on the device.

Every input of tests/test_animation_root_motion_cpu.py (each clip kind, length and bit width under every flag subset, on the root bone and
on a bone below it) is held bit for bit to the restatement (oracle_stack_rm, pinned to the reference-run vectors of
tests/golden/root_motion_kat.npz): absolute poses, dual quaternions and matrices at every lane count, in clip mode, clip mode with layers,
sample lists and stacks with IK.  Then: update_many over systems with and without root motion, the time step, calling twice, resetting,
and the refusals."""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from oracle import pyoracle as po
from oracle import pyrootmotion as prm
from bitexact import assert_bits_equal
from test_animation_root_motion_cpu import INPUTS, sample_plan

pytestmark = pytest.mark.gpu

DQ, MTX, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_MATRIX, lb.PALETTE_POSE
ALL = DQ | MTX | POSE
ERR_INVALID = lb._lib.ERR_INVALID
MODES = ("clips", "layers", "lists", "ik")
WEIGHTS = np.array([1.0, 0.99995, 0.9999, 0.99985, 0.5, 0.25], np.float32)


@pytest.fixture(scope="module")
def ctx():
    c = lb.Context(0)
    yield c
    c.close()


def _ik_chain(sk):
    """The deepest bone and the length of its root-to-leaf path."""
    depth = np.zeros(sk.bone_count, np.int64)
    for b in range(sk.bone_count):
        depth[b] = 0 if sk.parents[b] < 0 else depth[sk.parents[b]] + 1
    leaf = int(np.argmax(depth))
    return leaf, int(depth[leaf]) + 1


def plan(name, mode, seed=1):
    """The instances of one mode: (per-instance oracle stacks, a function that puts them into an AnimationSystem)."""
    sk, clips, bone, flags, tt, rt = INPUTS[name]
    rng = np.random.default_rng(seed)
    lengths = np.array([c.length_ticks for c in clips], np.int64)
    nc = len(clips)
    if mode in ("clips", "layers"):
        n = nc + 40
        ci = np.concatenate([np.arange(nc), rng.integers(0, nc, n - nc)]).astype(np.uint32)  # every clip at least once
        t = (rng.random(n) * lengths[ci]).astype(np.uint32)
        t[:8] = 0
        t[8:16] = lengths[ci[8:16]] - 1
        L = 2 if mode == "layers" else 0
        lc = rng.integers(0, nc, (n, L)).astype(np.uint32)
        lt = (rng.random((n, L)) * lengths[lc]).astype(np.uint32)
        lw = rng.choice(WEIGHTS, (n, L))
        stacks = [(np.r_[ci[i], lc[i]], np.r_[t[i], lt[i]], np.r_[np.float32(1), lw[i]], np.ones(L + 1, np.uint32), (), (), (), (), ()) for i in range(n)]

        def apply(a):
            a.setInstances(ci, t)
            if L:
                a.setLayers(lc, lt, lw)
        return stacks, apply, n
    n = 120
    counts = rng.integers(0, 5, n)
    counts[:4] = (0, 1, 1, 4)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    ci, t, w, lo = sample_plan(clips, int(offsets[-1]), seed=seed + 10)
    ik_counts = rng.integers(0, 3, n) if mode == "ik" else np.zeros(n, np.int64)
    ik_offsets = np.concatenate([[0], np.cumsum(ik_counts)]).astype(np.uint32)
    leaf, path = _ik_chain(sk)
    m = int(ik_offsets[-1])
    after = np.concatenate([np.sort(rng.integers(0, counts[i] + 1, ik_counts[i])) for i in range(n)]).astype(np.uint32) if m else np.zeros(0, np.uint32)
    leaves = np.full(m, leaf, np.uint32)
    bones = rng.integers(1, min(path, 4) + 1, m).astype(np.uint32)
    alpha = rng.choice(np.array([1.0, 0.7, 0.3], np.float32), m)
    target = (rng.normal(size=(m, 3)) * 0.5).astype(np.float32)
    stacks = []
    for i in range(n):
        s, e, a0, a1 = offsets[i], offsets[i + 1], ik_offsets[i], ik_offsets[i + 1]
        stacks.append((ci[s:e], t[s:e], w[s:e], lo[s:e], after[a0:a1], leaves[a0:a1], bones[a0:a1], alpha[a0:a1], target[a0:a1]))

    def apply(a):
        if mode == "ik":
            a.setStacks(offsets, ci, t, w, lo, ik_offsets, after, leaves, bones, alpha, target)
        else:
            a.setSamples(offsets, ci, t, w, lo)
    return stacks, apply, n


_EXPECTED = {}


def expected(name, mode, rm):
    key = (name, mode, None if rm is None else rm.tobytes())
    if key not in _EXPECTED:
        sk, clips = INPUTS[name][:2]
        stacks, _, n = plan(name, mode)
        B = sk.bone_count
        out = dict(pos=np.empty((n, B, 3), np.float32), rot=np.empty((n, B, 4), np.float32), dq=np.empty((n, B, 8), np.float32), mtx=np.empty((n, B, 16), np.float32))
        for i, s in enumerate(stacks):
            out["pos"][i], out["rot"][i] = prm.pose_stack(sk, clips, rm, *s)
            out["dq"][i], out["mtx"][i] = po.palettes(sk, out["pos"][i], out["rot"][i])
        _EXPECTED[key] = out
    return _EXPECTED[key]


def _rm(name):
    _, _, _, flags, tt, rt = INPUTS[name]
    return prm.root_motion(flags, tt, rt)


def _system(ctx, name, mode, rm=None, G=0):
    sk, clips = INPUTS[name][:2]
    _, apply, n = plan(name, mode)
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    a.setLaunch(G, 0)
    apply(a)
    if rm is not None:
        a.setRootMotion(rm["flags"], rm["translation_track"], rm["rotation_track"])
    return a


def _outputs(a):
    p, r = a.getPose()
    return dict(pos=p.copy(), rot=r.copy(), dq=a.getDualQuats().copy(), mtx=a.getMatrices().copy())


def _check(got, exp, what):
    for k in ("pos", "rot", "dq", "mtx"):
        assert_bits_equal(got[k], exp[k], f"{what}: {k}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(INPUTS))
@pytest.mark.parametrize("G", [4, 8, 16, 32])
def test_poses_equal_the_oracle(ctx, name, mode, G):
    rm = _rm(name)
    a = _system(ctx, name, mode, rm, G)
    a.update(0.0, ALL)
    assert a.lastLaunch()[0] == G
    _check(_outputs(a), expected(name, mode, rm), f"{name} {mode} G={G}")
    a.close()


def test_root_motion_changes_the_pose(ctx):
    """The inputs are not vacuous: with root motion the poses differ from the same system without it."""
    for name in INPUTS:
        with_rm, without = expected(name, "clips", _rm(name)), expected(name, "clips", None)
        assert not np.array_equal(with_rm["pos"].view(np.uint32), without["pos"].view(np.uint32)), name
        assert not np.array_equal(with_rm["rot"].view(np.uint32), without["rot"].view(np.uint32)), name


def test_time_stepping_is_unchanged(ctx):
    name = "root64"
    a, b = _system(ctx, name, "layers", _rm(name)), _system(ctx, name, "layers")
    for dt in (1.0 / 30.0, 0.4, -0.25, 0.0, 3.0):
        a.update(dt, ALL)
        b.update(dt, ALL)
        assert_bits_equal(a.getTimes(), b.getTimes(), f"times after a step of {dt}")
    a.close()
    b.close()


def test_update_many_mixed(ctx):
    """update_many over clip-mode, list and IK systems with and without root motion gives each system's own update."""
    def systems():
        return [_system(ctx, "root64", "clips", _rm("root64")), _system(ctx, "root64", "clips"), _system(ctx, "child64", "lists", _rm("child64")),
                _system(ctx, "child6", "ik", _rm("child6")), _system(ctx, "child6", "ik")]
    solo = systems()
    for s in solo:
        s.update(1.0 / 30.0, ALL)
    many = systems()
    lb.AnimationSystem.updateMany(many, 1.0 / 30.0, ALL)
    for k, (a, b) in enumerate(zip(solo, many)):
        _check(_outputs(b), _outputs(a), f"system {k}")
    for k in (0, 1):
        assert_bits_equal(many[k].getTimes(), solo[k].getTimes(), f"clip-mode times of system {k}")
    for s in solo + many:
        s.close()


def test_set_twice_and_reset(ctx):
    name = "child64"
    rm = _rm(name)
    a = _system(ctx, name, "lists", rm)
    a.setRootMotion(rm["flags"], rm["translation_track"], rm["rotation_track"])  # the same entries again
    a.update(0.0, ALL)
    _check(_outputs(a), expected(name, "lists", rm), "set twice")
    other = rm.copy()
    other["flags"] = (other["flags"] + 3) % 8  # a different flag set on every clip: replaces the first call
    a.setRootMotion(other["flags"], other["translation_track"], other["rotation_track"])
    a.update(0.0, ALL)
    _check(_outputs(a), expected(name, "lists", other), "a second, different call")
    a.setRootMotion(np.zeros(len(rm)), -1, -1)  # reset
    a.update(0.0, ALL)
    fresh = _system(ctx, name, "lists")
    fresh.update(0.0, ALL)
    _check(_outputs(a), _outputs(fresh), "reset against a system that never had root motion")
    a.setRootMotion(rm["flags"], rm["translation_track"], rm["rotation_track"])  # and back
    a.setRootMotion(rm["flags"], -1, -1)
    a.update(0.0, ALL)
    _check(_outputs(a), _outputs(fresh), "tracks -1 against a system that never had root motion")
    a.close()
    fresh.close()


def test_refusals_change_nothing(ctx):
    name = "child6"
    sk, clips, bone, flags, tt, rt = INPUTS[name]
    rm = _rm(name)
    a = _system(ctx, name, "ik", rm)
    a.update(0.0, ALL)
    exp = expected(name, "ik", rm)
    _check(_outputs(a), exp, "before the refusals")
    k = int(np.nonzero(tt >= 0)[0][0])

    def edit(field, v, i=k):
        r = rm.copy()
        r[field][i] = v
        return r

    refusals = {
        "flag bit 8": edit("flags", 8),
        "flags 0xffffffff": edit("flags", 0xffffffff),
        "translation track past the clip's": edit("translation_track", len(clips[k].translations)),
        "rotation track past the clip's": edit("rotation_track", len(clips[k].rotations)),
        "translation track -2": edit("translation_track", -2),
        "rotation track -2": edit("rotation_track", -2),
        "one entry too few": rm[:-1],
        "one entry too many": np.concatenate([rm, rm[:1]]),
        "no entries": rm[:0],
    }
    for what, r in refusals.items():
        with pytest.raises(lb.LumixB200Error) as e:
            a.setRootMotion(r["flags"], r["translation_track"], r["rotation_track"])
        assert e.value.code == ERR_INVALID, what
        a.update(0.0, ALL)
        _check(_outputs(a), exp, f"after the refusal '{what}'")
    assert a.L.lb200_animation_set_root_motion(a.h, C.c_uint32(len(clips)), None) == ERR_INVALID
    assert a.L.lb200_animation_set_root_motion(None, C.c_uint32(len(clips)), rm.ctypes.data_as(C.c_void_p)) == ERR_INVALID
    a.update(0.0, ALL)
    _check(_outputs(a), exp, "after the NULL refusals")
    a.close()
