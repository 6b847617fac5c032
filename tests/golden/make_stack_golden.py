"""Generates tests/golden/stack_kat.npz from the REFERENCE'S OWN getPose / evalBlendStack (controller.cpp:142-157, 267-293), cut out of
controller.cpp at build time into oracle/_ref/libanimation_shim_b200.so (oracle/build_ref.py; entry ref_pose_stack).  Run in
the build container only:  python tests/golden/make_stack_golden.py

Each stack is the bind pose + its SAMPLE instructions + Pose::computeAbsolute, on the skeletons and clips of stack_kat_inputs
(tests/test_animation_stacks_cpu.py rebuilds them from the same seeds and replays the stacks against oracle/oracle_stack.c)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from lumixengine_b200._lib import Clip  # noqa: E402  (the clip struct the animation harnesses take: stream byte counts included)
from oracle import pyoracle as po  # noqa: E402
from test_animation_stacks_cpu import stack_kat_inputs  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def stack_kat():
    L = C.CDLL(po.ANIMATION_SHIM_SO)
    d = {}
    for B, (sk, clips, cases) in stack_kat_inputs().items():
        arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
        rsk = po._skeleton_struct(sk, po.RefSkeleton)
        for k, (slot, weight, time_ticks, looped) in enumerate(cases):
            pos = np.zeros((B, 3), np.float32)
            rot = np.zeros((B, 4), np.float32)
            assert L.ref_pose_stack(C.byref(rsk), arr, C.c_uint32(len(clips)), po._ptr(slot), po._ptr(weight), po._ptr(time_ticks), po._ptr(looped),
                                    C.c_uint32(len(slot)), po._ptr(pos), po._ptr(rot)) == 0
            d[f"b{B}_c{k}_pos"], d[f"b{B}_c{k}_rot"] = pos, rot
    np.savez_compressed(os.path.join(OUT, "stack_kat.npz"), **d)
    print("stack_kat", len(d) // 2, "stacks")


if __name__ == "__main__":
    stack_kat()
