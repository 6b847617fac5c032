"""ctypes wrapper of oracle/liboracle_ik.so (oracle_ik.c): the IK instructions of an animator's blend stack, with its SAMPLE instructions,
restated on the CPU.  Types and helpers are pyoracle's; oracle/Makefile builds the library (lib() runs make)."""
import ctypes as C

import numpy as np

from . import pyoracle as po

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(po.make("liboracle_ik.so"))
    return _lib


def pose_stack_ik(skeleton, clips, clip, time_ticks, weight, looped, ik_after, ik_leaf, ik_bones, ik_alpha, ik_target):
    """pose_stack with IK instructions (evalIK, controller.cpp:159-265): op k runs on the relative pose after the first ik_after[k]
    samples, ops with the same ik_after in list order -> absolute (pos [B, 3], rot [B, 4])."""
    sk = po._skeleton_struct(skeleton, po.Skeleton)
    arr = (po.Clip * max(1, len(clips)))(*[c.as_struct(po.Clip) for c in clips])
    c = np.ascontiguousarray(clip, np.uint32)
    t = np.ascontiguousarray(time_ticks, np.uint32)
    w = np.ascontiguousarray(weight, np.float32)
    lo = np.ascontiguousarray(looped, np.uint32)
    assert len(c) == len(t) == len(w) == len(lo)
    ia = np.ascontiguousarray(ik_after, np.uint32)
    il = np.ascontiguousarray(ik_leaf, np.uint32)
    ib = np.ascontiguousarray(ik_bones, np.uint32)
    ial = np.ascontiguousarray(ik_alpha, np.float32)
    it = np.ascontiguousarray(np.asarray(ik_target, np.float32).reshape(-1, 3))
    assert len(ia) == len(il) == len(ib) == len(ial) == len(it)
    assert np.all(np.diff(ia.astype(np.int64)) >= 0) and (len(ia) == 0 or ia[-1] <= len(c))
    B = skeleton.bone_count
    pos = np.empty((B, 3), np.float32)
    rot = np.empty((B, 4), np.float32)
    lib().oracle_pose_stack_ik(C.byref(sk), arr, po._ptr(c), po._ptr(t), po._ptr(w), po._ptr(lo), C.c_uint32(len(c)), po._ptr(ia), po._ptr(il), po._ptr(ib),
                               po._ptr(ial), po._ptr(it), C.c_uint32(len(ia)), po._ptr(pos), po._ptr(rot))
    return pos, rot
