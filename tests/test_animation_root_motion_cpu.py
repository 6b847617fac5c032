"""Root motion in the pose path (Animation::setRootMotionBone, animation.cpp:214-270, and the sampling of the tracks it replaced) restated
on the CPU (oracle/oracle_root_motion.c).

The inputs are shared with tests/test_animation_root_motion_gpu.py and tests/golden/make_root_motion_golden.py: clips whose root-motion
bone (the root bone, or a bone below it) has a translation track, a rotation track, both or only constant tracks, at bit widths 5 to 16,
one frame long or hundreds of frames long, each under every subset of the root-motion flags."""
import ctypes as C
import os

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from lumixengine_b200.animation import AnimationClip
from oracle import pyoracle as po
from oracle import pyrootmotion as prm
from oracle import pystack

from bitexact import assert_bits_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KAT = os.path.join(ROOT, "tests", "golden", "root_motion_kat.npz")
SHIM = po.ANIMATION_SHIM_SO
FLAG_SETS = list(range(8))  # every subset of Y_ROOT_TRANSLATION | XZ_ROOT_TRANSLATION | ROOT_ROTATION
KINDS = ("both", "translation", "rotation", "constant")


def _yaw_quat(angle, tilt):
    """Unit quaternions (xyzw) of a yaw `angle` about Y followed by a small tilt about X, per frame."""
    h, t = angle * 0.5, tilt * 0.5
    qy = np.stack([np.zeros_like(h), np.sin(h), np.zeros_like(h), np.cos(h)], -1)
    qx = np.stack([np.sin(t), np.zeros_like(t), np.zeros_like(t), np.cos(t)], -1)
    x1, y1, z1, w1 = np.moveaxis(qy, -1, 0)
    x2, y2, z2, w2 = np.moveaxis(qx, -1, 0)
    q = np.stack([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2,
                  w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2], -1)
    return (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)


def rm_clip(sk, bone, kind, frames, pos_bits, rot_bits, seed):
    """A clip in which `bone` walks (translation: forward in XZ and bouncing in Y) and turns (rotation: yaw with a little tilt) as `kind`
    says, every other bone moves at random around the bind pose; tracks that never change are constant tracks (AnimationClip.encode)."""
    rng = np.random.default_rng(seed)
    B, n = sk.bone_count, frames + 1
    t = np.linspace(0.0, 1.0, n)[:, None]
    base_p, base_r = sk.bind_relative7[:, :3].astype(np.float64), sk.bind_relative7[:, 3:].astype(np.float64)
    pos = base_p[None] + 0.1 * rng.random((1, B, 3)) * np.sin(6.0 * t[..., None] + rng.random((1, B, 3)) * 6.0)
    rot = base_r[None] + 0.3 * rng.normal(size=(1, B, 4)) * np.sin(4.0 * t[..., None] + rng.random((1, B, 1)) * 6.0)
    rot = rot / np.linalg.norm(rot, axis=-1, keepdims=True)
    if kind in ("both", "translation"):
        pos[:, bone] = np.concatenate([1.5 * t, 0.05 + 0.1 * np.abs(np.sin(9.0 * t)), -2.5 * t + 0.3 * np.sin(3.0 * t)], 1)
    else:
        pos[:, bone] = pos[0, bone]
    if kind in ("both", "rotation"):
        rot[:, bone] = _yaw_quat(rng.uniform(-1, 1) + 2.8 * t[:, 0] * (1 if seed % 2 else -1), 0.15 * np.sin(5.0 * t[:, 0]))
    else:
        rot[:, bone] = rot[0, bone]
    return AnimationClip.encode(30.0, pos.astype(np.float32), rot.astype(np.float32), pos_bits=pos_bits, rot_bits=rot_bits)


def _skeleton_small():
    return scenes.skeleton(parents=[-1, 0, 1, 1, 3, 0])


def root_motion_inputs():
    """name -> (skeleton, clips, root-motion bone, per-clip flags, per-clip translation tracks, per-clip rotation tracks).  Each
    (kind, length, bit width) clip appears once per flag set, so one system holds every flag subset."""
    out = {}
    widths = [((5, 9, 16), (5, 7, 9)), ((12, 12, 12), (15, 15, 15)), ((16, 16, 16), (16, 11, 8)), ((8, 6, 10), (10, 13, 5))]
    for name, sk, bone in (("root64", scenes.skeleton(64), 0), ("child64", scenes.skeleton(64), 5), ("child6", _skeleton_small(), 3)):
        clips, flags = [], []
        for k, kind in enumerate(KINDS):
            for frames in (1, 7, 240):
                pb, rb = widths[(k + frames) % len(widths)]
                c = rm_clip(sk, bone, kind, frames, pb, rb, seed=17 * k + frames)
                for f in FLAG_SETS:
                    clips.append(c)
                    flags.append(f)
        tr = np.array([c.rootMotionTracks(bone) for c in clips], np.int32).reshape(-1, 2)
        out[name] = (sk, clips, bone, np.array(flags, np.uint32), tr[:, 0].copy(), tr[:, 1].copy())
    return out


def sample_plan(clips, n, seed):
    """n random (clip, time in ticks, weight, looped) samples over `clips`: times inside and past the clip, weights on both sides of
    0.9999."""
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    lengths = np.array([c.length_ticks for c in clips], np.int64)[ci]
    t = (rng.random(n) * lengths * 1.3).astype(np.uint32)
    w = rng.choice(np.array([1.0, 0.99995, 0.9999, 0.99985, 0.5, 0.25], np.float32), n)
    lo = rng.integers(0, 2, n).astype(np.uint32)
    return ci, t, w, lo


def pose_cases(clips, seed):
    """The sample stacks the fixture pins per input: 1 to 3 samples each."""
    rng = np.random.default_rng(seed)
    return [sample_plan(clips, int(rng.integers(1, 4)), seed=seed * 100 + k) for k in range(24)]


def math_inputs():
    """normalize(Quat) inputs: random quaternions at three scales, and the (0, y, 0, w) forms maskRootMotion normalises."""
    rng = np.random.default_rng(11)
    q = rng.normal(size=(4096, 4)).astype(np.float32) * rng.choice(np.array([1e-3, 1, 1e3], np.float32), (4096, 1))
    q[:8] = [[0, 1, 0, 0], [0, 0, 0, 1], [0, -0.0, 0, 1], [0, 0.6, 0, 0.8], [0, 1e-20, 0, 1e-20], [0, -3, 0, 4], [0, 0.5, 0, -0.5], [0, 0, 0, -1]]
    q[8:1024, 0] = 0
    q[8:1024, 2] = 0
    return q


def rotation_inputs(name):
    """(clip index, rotation track) pairs whose every frame Animation::getRotation is pinned for: the root-motion bone's track and track 0
    of every eighth clip of the input."""
    sk, clips, bone, flags, tt, rt = INPUTS[name]
    out = []
    for c in range(0, len(clips), 8):
        for r in sorted({0, int(rt[c])}):
            if 0 <= r < len(clips[c].rotations):
                out.append((c, r))
    return out


def run_ref_tables(L, clip, flags, bone):
    """setRootMotionBone through the reference harness -> (translation track, rotation track, pose_translations, pose_rotations)."""
    n = clip.frame_count + 1
    pt, pr, out3 = np.zeros((n, 3), np.float32), np.zeros((n, 4), np.float32), np.zeros(3, np.int32)
    cs = clip.as_struct(Clip)
    assert L.ref_rm_tables(C.byref(cs), C.c_uint32(flags), C.c_uint32(bone), po._ptr(pt), po._ptr(pr), po._ptr(out3)) == 0
    assert out3[2] in (0, n)
    return int(out3[0]), int(out3[1]), pt[:out3[2]], pr[:out3[2]]


def run_ref_pose_stack(L, sk, clips, flags, bone, ci, t, w, lo):
    B = sk.bone_count
    pos, rot = np.zeros((B, 3), np.float32), np.zeros((B, 4), np.float32)
    arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    rsk = po._skeleton_struct(sk, po.RefSkeleton)
    P = po._ptr
    assert L.ref_rm_pose_stack(C.byref(rsk), arr, P(np.ascontiguousarray(flags, np.uint32)), C.c_uint32(len(clips)), C.c_uint32(bone),
                               P(np.ascontiguousarray(ci, np.uint32)), P(np.ascontiguousarray(w, np.float32)), P(np.ascontiguousarray(t, np.uint32)),
                               P(np.ascontiguousarray(lo, np.uint32)), C.c_uint32(len(ci)), P(pos), P(rot)) == 0
    return pos, rot


def run_ref_math(L, q, clip=None, track=0):
    """normalize(Quat) of q, and Animation::getRotation of every frame of `track` of `clip`."""
    q = np.ascontiguousarray(q, np.float32)
    out = np.zeros_like(q)
    frames = np.arange(clip.frame_count + 1, dtype=np.uint32) if clip is not None else np.zeros(0, np.uint32)
    rot = np.zeros((len(frames), 4), np.float32)
    cs = clip.as_struct(Clip) if clip is not None else None
    assert L.ref_rm_math(po._ptr(q), C.c_uint32(len(q)), po._ptr(out), C.byref(cs) if cs is not None else None, C.c_uint32(track), po._ptr(frames),
                         C.c_uint32(len(frames)), po._ptr(rot)) == 0
    return out, rot


INPUTS = root_motion_inputs()


def test_every_case_is_covered():
    for name, (sk, clips, bone, flags, tt, rt) in INPUTS.items():
        assert set(flags.tolist()) == set(FLAG_SETS), name
        assert {(t >= 0, r >= 0) for t, r in zip(tt, rt)} == {(True, True), (True, False), (False, True), (False, False)}, name
        assert min(c.frame_count for c in clips) == 1 and max(c.frame_count for c in clips) >= 200, name
        bits = set(np.concatenate([np.concatenate([c.translations["bitsizes"].ravel(), c.rotations["bitsizes"].ravel()]) for c in clips]).tolist())
        assert min(bits) == 5 and max(bits) == 16, name
    assert {INPUTS[n][2] for n in INPUTS} >= {0, 5}  # the root bone and a bone below it


def test_without_root_motion_the_restatement_is_the_plain_one():
    """flags 0, or both tracks -1, leave the clip to its packed tracks: the same bytes as the blend-stack restatement."""
    for name, (sk, clips, bone, flags, tt, rt) in INPUTS.items():
        ci, t, w, lo = sample_plan(clips, 6, seed=3)
        want = pystack.pose_stack(sk, clips, ci, t, w, lo)
        for rm in (prm.root_motion(np.zeros(len(clips)), tt, rt), prm.root_motion(np.full(len(clips), 7), -1, -1), None):
            got = prm.pose_stack(sk, clips, rm, ci, t, w, lo)
            assert_bits_equal(got[0], want[0], f"{name}: positions")
            assert_bits_equal(got[1], want[1], f"{name}: rotations")


def test_flags_zero_returns_early():
    """setRootMotionBone returns before touching the clip when no root-motion flag is set (animation.cpp:216)."""
    sk, clips, bone, flags, tt, rt = INPUTS["root64"]
    for c, f, t, r in zip(clips, flags, tt, rt):
        ok, _, _ = prm.tables(c, int(f), int(t), int(r))
        assert ok == (f != 0)


def _kat():
    if not os.path.exists(KAT):
        pytest.skip("tests/golden/root_motion_kat.npz not present")
    return np.load(KAT)


def test_tables_equal_the_reference_vectors():
    kat = _kat()
    for name, (sk, clips, bone, flags, tt, rt) in INPUTS.items():
        assert_bits_equal(np.stack([tt, rt], 1), kat[f"{name}_tracks"], f"{name}: the tracks setRootMotionBone found (AnimationClip.rootMotionTracks)")
        for c, (clip, f, t, r) in enumerate(zip(clips, flags, tt, rt)):
            ok, pt, pr = prm.tables(clip, int(f), int(t), int(r))
            if not ok:
                continue
            assert_bits_equal(pt, kat[f"{name}_k{c}_pose_t"], f"{name} clip {c}: pose_translations")
            assert_bits_equal(pr, kat[f"{name}_k{c}_pose_r"], f"{name} clip {c}: pose_rotations")


def test_poses_equal_the_reference_vectors():
    kat = _kat()
    for name, (sk, clips, bone, flags, tt, rt) in INPUTS.items():
        rm = prm.root_motion(flags, tt, rt)
        for k in range(int(kat[f"{name}_n_cases"])):
            ci, t, w, lo = (kat[f"{name}_s{k}_{x}"] for x in ("clip", "time", "weight", "looped"))
            got = prm.pose_stack(sk, clips, rm, ci, t, w, lo)
            assert_bits_equal(got[0], kat[f"{name}_s{k}_pos"], f"{name} case {k}: positions")
            assert_bits_equal(got[1], kat[f"{name}_s{k}_rot"], f"{name} case {k}: rotations")


def test_math_helpers_on_the_host():
    """normalize(Quat) and the double-path Animation::getRotation of lb200_math.cuh, compiled for the host with the reference's flags,
    against the restatement (and, through the fixture, the reference)."""
    import subprocess
    import tempfile
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not installed")
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "rm_math.so")
        subprocess.check_call(["/usr/bin/g++", "-x", "c++", "-std=c++17", "-O2", "-msse2", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc,
                               "-I", os.path.join(ROOT, "lumixengine_b200", "csrc"), os.path.join(ROOT, "tests", "host_math", "root_motion_math_harness.cpp"), "-o", so])
        L = C.CDLL(so)
        q = math_inputs()
        got = np.empty_like(q)
        P = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
        L.rm_normalize(P(q), P(got), C.c_uint32(len(q)))
        assert_bits_equal(got, prm.quat_normalize(q), "normalize(Quat)")
        kat = np.load(KAT) if os.path.exists(KAT) else None
        if kat is not None:
            assert_bits_equal(got, kat["math_normalize"], "normalize(Quat) against the reference")
        for name, (sk, clips, *_rest) in INPUTS.items():
            for c, r in rotation_inputs(name):
                clip = clips[c]
                frames = np.arange(clip.frame_count + 1, dtype=np.uint32)
                tr = clip.rotations[r]
                mn, rng_, bits = (np.ascontiguousarray(tr[k], d) for k, d in (("min", np.float32), ("to_range", np.float32), ("bitsizes", np.uint32)))
                out = np.empty((len(frames), 4), np.float32)
                L.rm_rotation_d(P(clip.rotation_stream), C.c_uint32(clip.rotations_frame_size_bits), C.c_uint32(int(tr["offset_bits"])), P(mn), P(rng_), P(bits),
                                C.c_uint32(int(tr["skipped_channel"])), P(frames), P(out), C.c_uint32(len(frames)))
                assert_bits_equal(out, prm.rotation_d(clip, r, frames), f"{name} clip {c}: getRotation of track {r}")
                if kat is not None:
                    assert_bits_equal(out, kat[f"{name}_k{c}_rot{r}"], f"{name} clip {c}: getRotation of track {r} against the reference")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="root-motion harness not built (no reference tree where build() ran)")
def test_restatement_equals_reference_live():
    L = C.CDLL(SHIM)
    for name, (sk, clips, bone, flags, tt, rt) in INPUTS.items():
        rm = prm.root_motion(flags, tt, rt)
        for c, (clip, f) in enumerate(zip(clips, flags)):
            t, r, pt, pr = run_ref_tables(L, clip, int(f), bone)
            ok, ept, epr = prm.tables(clip, int(f), int(tt[c]), int(rt[c]))
            assert ok == (len(pt) > 0), f"{name} clip {c}"
            if ok:
                assert (t, r) == (tt[c], rt[c]), f"{name} clip {c}: tracks"
                assert_bits_equal(ept, pt, f"{name} clip {c}: pose_translations")
                assert_bits_equal(epr, pr, f"{name} clip {c}: pose_rotations")
        for k, (ci, t, w, lo) in enumerate(sample_plan(clips, 3, seed=500 + j) for j in range(6)):
            want = run_ref_pose_stack(L, sk, clips, flags, bone, ci, t, w, lo)
            got = prm.pose_stack(sk, clips, rm, ci, t, w, lo)
            assert_bits_equal(got[0], want[0], f"{name} stack {k}: positions")
            assert_bits_equal(got[1], want[1], f"{name} stack {k}: rotations")
