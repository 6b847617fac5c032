"""Generates tests/golden/ik_kat.npz from the REFERENCE'S OWN evalBlendStack / evalIK (controller.cpp:159-293) and math (Quat::vec3ToVec3,
nlerp, LocalRigidTransform::inverted, length, Quat::conjugated), cut out of the reference at build time into
oracle/_ref/libanimation_shim_b200.so (oracle/build_ref.py; entries ref_pose_stack_ik, ref_ik_math).  Run in the build
container only:  python tests/golden/make_ik_golden.py

Each stack is the bind pose + its SAMPLE and IK instructions in order + Pose::computeAbsolute, on a Model with a bone map, for the
skeletons, clips and cases of ik_kat_inputs (tests/test_animation_ik_cpu.py rebuilds them from the same seeds).  Cases whose reference
result holds a NaN are refused here: they are outside the bit-for-bit contract (DESIGN.md section 2)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pyoracle as po  # noqa: E402
from test_animation_ik_cpu import ik_kat_inputs, ik_math_inputs, run_ref_stack_ik  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def ik_kat():
    L = C.CDLL(po.ANIMATION_SHIM_SO)
    d = {}
    for name, (sk, clips, cases) in ik_kat_inputs().items():
        for k, case in enumerate(cases):
            pos, rot = run_ref_stack_ik(L, sk, clips, case)
            assert not (np.isnan(pos).any() or np.isnan(rot).any()), f"{name} case {k}: the reference computes a NaN"
            d[f"{name}_c{k}_pos"], d[f"{name}_c{k}_rot"] = pos, rot
    m = ik_math_inputs()
    n = len(m["v0"])
    outs = {"m_vec3_to_vec3": np.zeros((n, 4), np.float32), "m_nlerp": np.zeros((n, 4), np.float32), "m_inverted": np.zeros((n, 7), np.float32),
            "m_length": np.zeros(n, np.float32), "m_conjugated": np.zeros((n, 4), np.float32)}
    P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert L.ref_ik_math(C.c_uint32(n), P(m["v0"]), P(m["v1"]), P(m["qa"]), P(m["qb"]), P(m["t"]), P(m["lrt"]), P(outs["m_vec3_to_vec3"]),
                         P(outs["m_nlerp"]), P(outs["m_inverted"]), P(outs["m_length"]), P(outs["m_conjugated"])) == 0
    d.update({f"m_{k}": v for k, v in m.items()})
    d.update(outs)
    np.savez_compressed(os.path.join(OUT, "ik_kat.npz"), **d)
    print("ik_kat", sum(1 for f in d if f.endswith("_pos")), "stacks,", n, "math vectors")


if __name__ == "__main__":
    ik_kat()
