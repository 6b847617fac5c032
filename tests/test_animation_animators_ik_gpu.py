"""The animator binding (AnimatorsB200, host/animators_b200.inl) with IK instructions, over real Model / Animation / Pose objects whose
Models have a bone map (oracle/_ref/libanimation_shim_b200.so, entry ashim_run_animators_ik, built by oracle/build_ref.py where
the reference tree exists; skipped elsewhere).  Over several frames and three models, every pose must be bit-equal to the reference's
getRelativePose + evalBlendStack + computeAbsolute; IK animators stay off referencePath() unless an IK instruction's leaf bone is
missing, its bone count is 0 or above 32, or its chain leaves the skeleton (or the controller has bone masks); every animator gets one
lock and one unlock per frame."""
import ctypes as C
import os

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from oracle import pyoracle as po
from bitexact import assert_bits_equal
from test_animation_ik_cpu import depths

pytestmark = pytest.mark.gpu

SO = po.ANIMATION_SHIM_SO


@pytest.mark.skipif(not os.path.exists(SO), reason="animator harness not built (no reference tree where build() ran)")
def test_ik_animators_binding_equals_reference():
    L = C.CDLL(SO)
    sks = [scenes.skeleton(64, seed=4), scenes.skeleton(seed=40, parents=[-1] + list(range(0, 33)) + [3, 10, 20, 30, 33, 34]),
           scenes.skeleton(seed=1, parents=[-1])]
    clips, clip_start = [], [0]
    for m, sk in enumerate(sks):
        clips += [scenes.clip(sk, frames=13 + m, fps=30.0, seed=10 * m + 1, const_fraction=0.3), scenes.clip(sk, frames=40, fps=24.0, seed=10 * m + 2),
                  scenes.clip(sk, frames=7, fps=60.0, seed=10 * m + 3, const_fraction=0.5)]
        clip_start.append(len(clips))
    null_slot = np.full(3, 99, np.uint32)
    n_anim, n_frames = 48, 4
    rng = np.random.default_rng(9)
    model_of = rng.integers(0, 3, n_anim).astype(np.uint32)
    masked = np.zeros(n_anim, np.uint32)
    masked[7] = 1
    ctx_weight = np.where(np.arange(n_anim) % 4 == 1, 0.75, 1.0).astype(np.float32)
    d = [depths(sk.parents) for sk in sks]
    cols = {k: [] for k in ("kind", "slot", "weight", "time", "looped", "leaf", "bones", "alpha")}
    target = []
    instr_start, n_instr = [], []
    expect_ref = np.zeros((n_frames, n_anim), bool)
    for f in range(n_frames):
        for i in range(n_anim):
            m = int(model_of[i])
            B = sks[m].bone_count
            n_samples = [0, 1, 2, 3][(i + f) % 4]
            # IK ops: one or two, between the samples; every 9th animator's first op is one the binding must leave to the reference
            n_ik = 0 if i % 5 == 4 else 1 + (i + f) % 2
            after = np.sort(rng.integers(0, n_samples + 1, n_ik))
            bad = (i % 9 == 2) and n_ik > 0
            instr_start.append(len(cols["kind"]))
            s = k = 0
            count = 0
            while s <= n_samples:
                while k < n_ik and after[k] == s:
                    deep = np.nonzero(d[m] >= 1)[0]
                    leaf = int(deep[rng.integers(0, len(deep))]) if len(deep) else 0
                    bones = int(rng.integers(1, min(32, d[m][leaf] + 1) + 1))
                    alpha = [1.0, 0.5, 0.0, 0.001][(i + k) % 4]
                    if bad and k == 0:
                        # missing leaf, count 0, 33, chain off the root: the reference writes out of bounds or reads bone -1 for these
                        # unless alpha < 0.001 returns first (controller.cpp:167), the binding leaves them to it whatever the alpha
                        leaf, bones = [(B + 3, 2), (leaf, 0), (leaf, 33), (0, 2)][(i // 9 + f) % 4]
                        alpha = 0.0
                    cols["kind"].append(2)
                    for key, v in (("slot", 0), ("weight", 0.0), ("time", 0), ("looped", 0), ("leaf", leaf), ("bones", bones), ("alpha", alpha)):
                        cols[key].append(v)
                    target.append((sks[m].bind_abs7[0, :3] + rng.normal(size=3) * [0.3, 3.0][(i + k + f) % 2]).astype(np.float32))
                    k += 1
                    count += 1
                if s == n_samples:
                    break
                slot = int(rng.integers(0, 3))
                length = clips[clip_start[m] + slot].length_ticks
                cols["kind"].append(1)
                for key, v in (("slot", slot), ("weight", [1.0, 0.5, 0.25][int(rng.integers(0, 3))] if s else 1.0), ("time", int(rng.integers(0, 2 * length))),
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
    sk_arr = (po.RefSkeleton * 3)(*[po._skeleton_struct(s, po.RefSkeleton) for s in sks])
    clip_arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    bones = np.array([s.bone_count for s in sks])[model_of]
    total = int(bones.sum()) * n_frames
    pos_ref, pos_b = np.zeros((total, 3), np.float32), np.zeros((total, 3), np.float32)
    rot_ref, rot_b = np.zeros((total, 4), np.float32), np.zeros((total, 4), np.float32)
    on_ref = np.zeros(n_frames * n_anim, np.uint32)
    info = np.zeros(3, np.uint32)
    P = po._ptr
    rc = L.ashim_run_animators_ik(sk_arr, C.c_uint32(3), clip_arr, P(np.array(clip_start, np.uint32)), P(null_slot), P(model_of), P(masked), C.c_uint32(n_anim),
                                  C.c_uint32(n_frames), P(instr_start), P(n_instr), P(col["kind"]), P(col["slot"]), P(col["weight"]), P(col["time"]), P(col["looped"]),
                                  P(col["leaf"]), P(col["bones"]), P(col["alpha"]), P(tgt), P(ctx_weight),
                                  P(pos_ref), P(rot_ref), P(pos_b), P(rot_b), P(on_ref), P(info))
    assert rc == 0 and info[2] == 0, f"harness rc {rc}, binding rc {info[2]}"
    assert info[0] == 1 and info[1] == 1, f"locks / unlocks per animator and frame: max {info[0]}, min {info[1]}"
    assert np.array_equal(on_ref.reshape(n_frames, n_anim).astype(bool), expect_ref), "animators on the reference path"
    assert expect_ref.any() and (~expect_ref).sum() > n_anim
    assert_bits_equal(pos_b, pos_ref, "positions")
    assert_bits_equal(rot_b, rot_ref, "rotations")
