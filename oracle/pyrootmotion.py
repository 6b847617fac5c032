"""ctypes wrapper of oracle/liboracle_root_motion.so (oracle_root_motion.c): Animation::setRootMotionBone and the sampling of clips whose
root-motion tracks it replaced, restated on the CPU.  Types and helpers are pyoracle's; oracle/Makefile builds the
library (lib() runs make)."""
import ctypes as C

import numpy as np

from . import pyoracle as po

ROOT_MOTION_DTYPE = np.dtype([("flags", np.uint32), ("translation_track", np.int32), ("rotation_track", np.int32)])  # lb200_root_motion
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(po.make("liboracle_root_motion.so"))
    return _lib


def root_motion(flags, translation_track, rotation_track):
    """Per-clip entries in lb200_root_motion form."""
    rm = np.zeros(len(np.atleast_1d(flags)), ROOT_MOTION_DTYPE)
    rm["flags"], rm["translation_track"], rm["rotation_track"] = flags, translation_track, rotation_track
    return rm


def tables(clip, flags, translation_track, rotation_track):
    """setRootMotionBone (animation.cpp:214-270) on a freshly loaded clip -> (replaced, pose_translations [F+1, 3], pose_rotations [F+1, 4]);
    replaced is False when the call returns early (no root-motion flag)."""
    cs = clip.as_struct(po.Clip)
    n = clip.frame_count + 1
    pt = np.zeros((n, 3), np.float32)
    pr = np.zeros((n, 4), np.float32)
    ok = lib().oracle_root_motion_tables(C.byref(cs), C.c_uint32(flags), C.c_int32(translation_track), C.c_int32(rotation_track), po._ptr(pt), po._ptr(pr))
    return bool(ok), pt, pr


def pose_stack(skeleton, clips, rm, clip, time_ticks, weight, looped, ik_after=(), ik_leaf=(), ik_bones=(), ik_alpha=(), ik_target=()):
    """Bind pose + samples in order (getPose's time rule) with IK ops between them, over clips with root motion rm (root_motion(), one
    entry per clip, or None) + Pose::computeAbsolute -> absolute (pos [B, 3], rot [B, 4])."""
    sk = po._skeleton_struct(skeleton, po.Skeleton)
    arr = (po.Clip * max(1, len(clips)))(*[c.as_struct(po.Clip) for c in clips])
    rm = None if rm is None else np.ascontiguousarray(rm, ROOT_MOTION_DTYPE)
    assert rm is None or len(rm) == len(clips)
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
    rc = lib().oracle_stack_rm(C.byref(sk), arr, C.c_uint32(len(clips)), po._ptr(rm), po._ptr(c), po._ptr(t), po._ptr(w), po._ptr(lo), C.c_uint32(len(c)),
                               po._ptr(ia), po._ptr(il), po._ptr(ib), po._ptr(ial), po._ptr(it), C.c_uint32(len(ia)), po._ptr(pos), po._ptr(rot))
    assert rc == 0, "oracle_stack_rm: out of memory"
    return pos, rot


def quat_normalize(q):
    q = np.ascontiguousarray(q, np.float32).reshape(-1, 4)
    out = np.empty_like(q)
    lib().oracle_quat_normalize(po._ptr(q), po._ptr(out), C.c_uint32(len(q)))
    return out


def rotation_d(clip, track, frames):
    """Animation::getRotation (animation.cpp:336-364, unpackChannel through double) of rotation track `track` at each frame."""
    cs = clip.as_struct(po.Clip)
    f = np.ascontiguousarray(frames, np.uint32)
    out = np.empty((len(f), 4), np.float32)
    lib().oracle_rotation_d(C.byref(cs), C.c_uint32(track), po._ptr(f), po._ptr(out), C.c_uint32(len(f)))
    return out
