"""The animator binding (AnimatorsB200, host/animators_b200.inl) executed over real Model / Animation / Pose objects and scripted blend
stacks (oracle/_ref/libanimation_shim_b200.so, built by oracle/build_ref.py where the reference tree exists; skipped elsewhere).
Over several frames and three models, every pose must be bit-equal to the reference's getRelativePose + evalBlendStack + computeAbsolute;
animators with an IK instruction or a controller with bone masks must land on referencePath(); every animator gets one lock
and one unlock per frame."""
import ctypes as C
import os

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from oracle import pyoracle as po
from bitexact import assert_bits_equal

pytestmark = pytest.mark.gpu

SO = po.ANIMATION_SHIM_SO
BELOW = float(np.nextafter(np.float32(0.9999), np.float32(0)))


@pytest.mark.skipif(not os.path.exists(SO), reason="animator harness not built (no reference tree where build() ran)")
def test_animators_binding_equals_reference():
    L = C.CDLL(SO)
    sks = [scenes.skeleton(64, seed=4), scenes.skeleton(seed=20, parents=[-1] + [i // 2 for i in range(1, 20)]), scenes.skeleton(seed=1, parents=[-1])]
    clips, clip_start = [], [0]
    for m, sk in enumerate(sks):
        clips += [scenes.clip(sk, frames=13 + m, fps=30.0, seed=10 * m + 1, const_fraction=0.3), scenes.clip(sk, frames=40, fps=24.0, seed=10 * m + 2),
                  scenes.clip(sk, frames=7, fps=60.0, seed=10 * m + 3, const_fraction=0.5)]
        clip_start.append(len(clips))
    null_slot = np.full(3, 99, np.uint32)  # no null slot: the reference's getPose dereferences it (controller.cpp:144)
    n_anim, n_frames = 40, 4
    rng = np.random.default_rng(5)
    model_of = rng.integers(0, 3, n_anim).astype(np.uint32)
    masked = np.zeros(n_anim, np.uint32)
    masked[7] = 1
    cols = {k: [] for k in ("kind", "slot", "weight", "time", "looped")}
    instr_start, n_instr = [], []
    expect_ref = np.zeros((n_frames, n_anim), bool)
    for f in range(n_frames):
        for i in range(n_anim):
            n = [0, 1, 2, 3, 6][(i + f) % 5]
            instr_start.append(len(cols["kind"]))
            n_instr.append(n)
            has_ik = (i % 11 == 3) and n > 0
            for k in range(n):
                kind = 2 if has_ik and k == n - 1 else 1
                slot = int(rng.integers(0, 3))
                cols["kind"].append(kind)
                cols["slot"].append(slot)
                cols["weight"].append([0.0, BELOW, 0.9999, 1.0, 2.0, 0.5][int(rng.integers(0, 6))] if k else (1.0 if i % 2 else 0.4))
                length = clips[clip_start[model_of[i]] + slot].length_ticks
                cols["time"].append(int([0, length - 1, length, 3 * length + 5, rng.integers(0, length)][int(rng.integers(0, 5))]))
                cols["looped"].append(int(rng.integers(0, 2)))
            expect_ref[f, i] |= has_ik or bool(masked[i])
    col = {k: np.array(v, np.float32 if k == "weight" else np.uint32) for k, v in cols.items()}
    instr_start, n_instr = np.array(instr_start, np.uint32), np.array(n_instr, np.uint32)
    sk_arr = (po.RefSkeleton * 3)(*[po._skeleton_struct(s, po.RefSkeleton) for s in sks])
    clip_arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    bones = np.array([s.bone_count for s in sks])[model_of]
    total = int(bones.sum()) * n_frames
    pos_ref, pos_b = np.zeros((total, 3), np.float32), np.zeros((total, 3), np.float32)
    rot_ref, rot_b = np.zeros((total, 4), np.float32), np.zeros((total, 4), np.float32)
    on_ref = np.zeros(n_frames * n_anim, np.uint32)
    info = np.zeros(3, np.uint32)
    P = po._ptr
    rc = L.ashim_run_animators(sk_arr, C.c_uint32(3), clip_arr, P(np.array(clip_start, np.uint32)), P(null_slot), P(model_of), P(masked), C.c_uint32(n_anim),
                               C.c_uint32(n_frames), P(instr_start), P(n_instr), P(col["kind"]), P(col["slot"]), P(col["weight"]), P(col["time"]), P(col["looped"]),
                               P(pos_ref), P(rot_ref), P(pos_b), P(rot_b), P(on_ref), P(info))
    assert rc == 0 and info[2] == 0, f"harness rc {rc}, binding rc {info[2]}"
    assert info[0] == 1 and info[1] == 1, f"locks / unlocks per animator and frame: max {info[0]}, min {info[1]}"
    assert np.array_equal(on_ref.reshape(n_frames, n_anim).astype(bool), expect_ref), "animators on the reference path"
    assert expect_ref.any() and not expect_ref.all()
    assert_bits_equal(pos_b, pos_ref, "positions")
    assert_bits_equal(rot_b, rot_ref, "rotations")
