"""ctypes wrapper of oracle/liboracle_stack.so (oracle_stack.c): the SAMPLE instructions of an animator's blend stack restated on the CPU.
Types and helpers are pyoracle's; oracle/Makefile builds the library (lib() runs make)."""
import ctypes as C

import numpy as np

from . import pyoracle as po

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(po.make("liboracle_stack.so"))
    return _lib


def pose_stack(skeleton, clips, clip, time_ticks, weight, looped):
    """Bind pose + one animator's SAMPLE instructions in order (evalBlendStack / getPose, controller.cpp:142-157, 267-293) +
    Pose::computeAbsolute -> absolute (pos [B, 3], rot [B, 4])."""
    sk = po._skeleton_struct(skeleton, po.Skeleton)
    arr = (po.Clip * len(clips))(*[c.as_struct(po.Clip) for c in clips])
    c = np.ascontiguousarray(clip, np.uint32)
    t = np.ascontiguousarray(time_ticks, np.uint32)
    w = np.ascontiguousarray(weight, np.float32)
    lo = np.ascontiguousarray(looped, np.uint32)
    assert len(c) == len(t) == len(w) == len(lo)
    B = skeleton.bone_count
    pos = np.empty((B, 3), np.float32)
    rot = np.empty((B, 4), np.float32)
    lib().oracle_pose_stack(C.byref(sk), arr, po._ptr(c), po._ptr(t), po._ptr(w), po._ptr(lo), C.c_uint32(len(c)), po._ptr(pos), po._ptr(rot))
    return pos, rot
