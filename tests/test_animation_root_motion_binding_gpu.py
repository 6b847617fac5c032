"""The engine bindings (AnimablesB200, AnimatorsB200) over real Animation objects whose root motion the reference's own
Animation::setRootMotionBone set (oracle/_ref/libanimation_shim_b200.so, entries ashim_run_animables_rm / ashim_run_animators_rm, built
by oracle/build_ref.py where the reference tree exists; skipped elsewhere).  Over several frames every pose (and animable
time) must be bit-equal to the reference's updateAnimable / evalBlendStack; AnimablesB200 poses every animable itself, animators with
root-motion clips stay off AnimatorsB200::referencePath() while bone masks and unresolvable IK instructions still go there; every entity
gets one lock and one unlock per frame."""
import ctypes as C
import os

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from oracle import pyoracle as po
from bitexact import assert_bits_equal
from test_animation_ik_cpu import depths
from test_animation_root_motion_cpu import INPUTS, rm_clip

pytestmark = pytest.mark.gpu

SO = po.ANIMATION_SHIM_SO
needs_shim = pytest.mark.skipif(not os.path.exists(SO), reason="root-motion harness not built (no reference tree where build() ran)")
P = po._ptr


@needs_shim
@pytest.mark.parametrize("name", list(INPUTS))
def test_animables_binding_equals_reference(name):
    L = C.CDLL(SO)
    sk, clips, bone, flags, tt, rt = INPUTS[name]
    n_inst, rounds, B = 2 * len(clips), 4, sk.bone_count
    rng = np.random.default_rng(3)
    ci = np.concatenate([np.arange(len(clips)), rng.integers(0, len(clips), n_inst - len(clips))]).astype(np.uint32)
    tt0 = (rng.random(n_inst) * np.array([c.length_ticks for c in clips])[ci]).astype(np.uint32)
    arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    rsk = po._skeleton_struct(sk, po.RefSkeleton)
    out = {k: np.zeros((rounds, n_inst, B, w), np.float32) for k, w in (("pos_ref", 3), ("rot_ref", 4), ("pos_b", 3), ("rot_b", 4))}
    t_ref, t_b = np.zeros((rounds, n_inst), np.uint32), np.zeros((rounds, n_inst), np.uint32)
    info = np.zeros(3, np.uint32)
    rc = L.ashim_run_animables_rm(C.byref(rsk), arr, P(flags), C.c_uint32(len(clips)), C.c_uint32(bone), P(ci), P(tt0), C.c_uint32(n_inst),
                                  C.c_float(1.0 / 30.0), C.c_uint32(rounds), P(out["pos_ref"]), P(out["rot_ref"]), P(t_ref), P(out["pos_b"]),
                                  P(out["rot_b"]), P(t_b), P(info))
    assert rc == 0 and info[2] == 0, f"harness rc {rc}, binding rc {info[2]}"
    assert info[0] == info[1] == n_inst * rounds, f"locks {info[0]}, unlocks {info[1]} for {n_inst} animables x {rounds} frames"
    for f in range(rounds):
        assert_bits_equal(out["pos_b"][f], out["pos_ref"][f], f"{name} frame {f}: positions")
        assert_bits_equal(out["rot_b"][f], out["rot_ref"][f], f"{name} frame {f}: rotations")
        assert_bits_equal(t_b[f], t_ref[f], f"{name} frame {f}: times")


@needs_shim
def test_animators_binding_equals_reference():
    L = C.CDLL(SO)
    bone = 3
    sks = [scenes.skeleton(64, seed=4), scenes.skeleton(parents=[-1, 0, 1, 1, 3, 0])]
    plan = [("both", 7, 1), ("translation", 1, 9), ("rotation", 4, 30), ("both", 2, 17), ("constant", 7, 5), ("both", 0, 12), ("translation", 3, 60),
            ("rotation", 5, 3)]
    clips, flags, clip_start = [], [], [0]
    for m, sk in enumerate(sks):
        for j, (kind, f, frames) in enumerate(plan):
            clips.append(rm_clip(sk, bone, kind, frames, (11, 9, 14), (13, 12, 10), seed=100 * m + j))
            flags.append(f)
        clip_start.append(len(clips))
    flags = np.array(flags, np.uint32)
    assert any(clips[c].rootMotionTracks(bone) != (-1, -1) and flags[c] for c in range(len(clips)))
    null_slot = np.full(len(sks), 99, np.uint32)
    n_anim, n_frames = 40, 4
    rng = np.random.default_rng(21)
    model_of = rng.integers(0, len(sks), n_anim).astype(np.uint32)
    masked = np.zeros(n_anim, np.uint32)
    masked[7] = 1
    d = [depths(sk.parents) for sk in sks]
    cols = {k: [] for k in ("kind", "slot", "weight", "time", "looped", "leaf", "bones", "alpha")}
    target, instr_start, n_instr = [], [], []
    expect_ref = np.zeros((n_frames, n_anim), bool)
    n_slots = len(plan)
    for f in range(n_frames):
        for i in range(n_anim):
            m = int(model_of[i])
            B = sks[m].bone_count
            n_samples = [1, 2, 3, 0][(i + f) % 4]
            n_ik = 1 if i % 3 == 0 else 0
            after = np.sort(rng.integers(0, n_samples + 1, n_ik))
            bad = (i % 9 == 3) and n_ik > 0  # an IK leaf the model does not name: left to the reference
            instr_start.append(len(cols["kind"]))
            s = k = count = 0
            while s <= n_samples:
                while k < n_ik and after[k] == s:
                    deep = np.nonzero(d[m] >= 1)[0]
                    leaf = int(deep[rng.integers(0, len(deep))])
                    leaf, bones = (B + 3, 2) if bad else (leaf, int(rng.integers(1, d[m][leaf] + 2)))
                    cols["kind"].append(2)
                    for key, v in (("slot", 0), ("weight", 0.0), ("time", 0), ("looped", 0), ("leaf", leaf), ("bones", bones), ("alpha", 0.0 if bad else 0.8)):
                        cols[key].append(v)
                    target.append((sks[m].bind_abs7[0, :3] + rng.normal(size=3) * 0.5).astype(np.float32))
                    k += 1
                    count += 1
                if s == n_samples:
                    break
                slot = int(rng.integers(0, n_slots))
                length = clips[clip_start[m] + slot].length_ticks
                cols["kind"].append(1)
                for key, v in (("slot", slot), ("weight", [1.0, 0.5, 0.99995][int(rng.integers(0, 3))] if s else 1.0), ("time", int(rng.integers(0, 2 * length))),
                               ("looped", int(rng.integers(0, 2))), ("leaf", 0), ("bones", 0), ("alpha", 0.0)):
                    cols[key].append(v)
                target.append(np.zeros(3, np.float32))
                s += 1
                count += 1
            n_instr.append(count)
            expect_ref[f, i] = bad or bool(masked[i])
    col = {k: np.array(v, np.float32 if k in ("weight", "alpha") else np.uint32) for k, v in cols.items()}
    tgt = np.ascontiguousarray(np.array(target, np.float32).reshape(-1, 3))
    instr_start, n_instr = np.array(instr_start, np.uint32), np.array(n_instr, np.uint32)
    sk_arr = (po.RefSkeleton * len(sks))(*[po._skeleton_struct(s, po.RefSkeleton) for s in sks])
    clip_arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    total = int(np.array([s.bone_count for s in sks])[model_of].sum()) * n_frames
    pos_ref, pos_b = np.zeros((total, 3), np.float32), np.zeros((total, 3), np.float32)
    rot_ref, rot_b = np.zeros((total, 4), np.float32), np.zeros((total, 4), np.float32)
    on_ref, info = np.zeros(n_frames * n_anim, np.uint32), np.zeros(3, np.uint32)
    rc = L.ashim_run_animators_rm(sk_arr, C.c_uint32(len(sks)), clip_arr, P(flags), C.c_uint32(bone), P(np.array(clip_start, np.uint32)), P(null_slot),
                                  P(model_of), P(masked), C.c_uint32(n_anim), C.c_uint32(n_frames), P(instr_start), P(n_instr), P(col["kind"]), P(col["slot"]),
                                  P(col["weight"]), P(col["time"]), P(col["looped"]), P(col["leaf"]), P(col["bones"]), P(col["alpha"]), P(tgt),
                                  P(pos_ref), P(rot_ref), P(pos_b), P(rot_b), P(on_ref), P(info))
    assert rc == 0 and info[2] == 0, f"harness rc {rc}, binding rc {info[2]}"
    assert info[0] == 1 and info[1] == 1, f"locks / unlocks per animator and frame: max {info[0]}, min {info[1]}"
    assert np.array_equal(on_ref.reshape(n_frames, n_anim).astype(bool), expect_ref), "animators on the reference path"
    assert expect_ref.any() and (~expect_ref).sum() > n_anim
    assert_bits_equal(pos_b, pos_ref, "positions")
    assert_bits_equal(rot_b, rot_ref, "rotations")
