"""Generates tests/golden/root_motion_kat.npz from the REFERENCE'S OWN Animation::setRootMotionBone, Animation::getRotation, normalize(Quat)
and, for whole poses, Model::getRelativePose + evalBlendStack + Pose::computeAbsolute over Animation objects whose root motion
setRootMotionBone set (oracle/_ref/libanimation_shim_b200.so, built by oracle/build_ref.py; entries ref_rm_tables,
ref_rm_pose_stack, ref_rm_math).  Run in the build container only:  python tests/golden/make_root_motion_golden.py

The inputs are root_motion_inputs (tests/test_animation_root_motion_cpu.py rebuilds them from the same seeds): per input, the tracks
setRootMotionBone found, the pose_translations / pose_rotations of every clip whose flags are not 0, 24 sample stacks (pose_cases) and
getRotation of every frame of the tracks rotation_inputs names; then normalize(Quat) of math_inputs."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pyoracle as po  # noqa: E402
from test_animation_root_motion_cpu import (INPUTS, math_inputs, pose_cases, rotation_inputs, run_ref_math, run_ref_pose_stack,  # noqa: E402
                                            run_ref_tables)

OUT = os.path.dirname(os.path.abspath(__file__))


def root_motion_kat():
    L = C.CDLL(po.ANIMATION_SHIM_SO)
    d = {}
    for s_idx, (name, (sk, clips, bone, flags, tt, rt)) in enumerate(INPUTS.items()):
        tracks = np.zeros((len(clips), 2), np.int32)
        for c, (clip, f) in enumerate(zip(clips, flags)):
            t, r, pt, pr = run_ref_tables(L, clip, int(f), bone)
            tracks[c] = (t, r) if f else (tt[c], rt[c])  # with flags 0 the reference returns before it looks the tracks up
            if len(pt):
                d[f"{name}_k{c}_pose_t"], d[f"{name}_k{c}_pose_r"] = pt, pr
        d[f"{name}_tracks"] = tracks
        cases = pose_cases(clips, seed=s_idx + 1)
        d[f"{name}_n_cases"] = np.array(len(cases))
        for k, (ci, t, w, lo) in enumerate(cases):
            d[f"{name}_s{k}_clip"], d[f"{name}_s{k}_time"], d[f"{name}_s{k}_weight"], d[f"{name}_s{k}_looped"] = ci, t, w, lo
            d[f"{name}_s{k}_pos"], d[f"{name}_s{k}_rot"] = run_ref_pose_stack(L, sk, clips, flags, bone, ci, t, w, lo)
        for c, r in rotation_inputs(name):
            d[f"{name}_k{c}_rot{r}"] = run_ref_math(L, np.zeros((0, 4), np.float32), clips[c], r)[1]
    d["math_normalize"] = run_ref_math(L, math_inputs())[0]
    np.savez_compressed(os.path.join(OUT, "root_motion_kat.npz"), **d)
    print("root_motion_kat", sum(1 for k in d if k.endswith("_pose_t")), "tables,", sum(1 for k in d if k.endswith("_pos")), "stacks")


if __name__ == "__main__":
    root_motion_kat()
