"""Clips at the edges the importer can reach and the narrow synthetic clips of the other tests do not: long clips (up to 4097 frames) at
and past their end, and every channel width, from raw bit streams rather than AnimationClip.encode.

The inputs are shared with tests/test_animation_clip_edges_gpu.py:
  LENGTH_CLIPS  frame counts 1, 2, 255, 256, 257, 300, 1000 and 4097 at 1, 24, 25, 30, 59.94 and 60 fps on a six-bone skeleton
  WIDTH_CLIPS   one clip per translation width set on a 64-bone skeleton: every width 1 .. 32 in each channel, (32, 32, 32), (31, 31, 31)
                and channels of 33 to 63 bits; rotation widths the importer's clampBitsizes allows and wider ones for the 64-bit path
Every stream is random bytes, exactly (frame_count + 1) frames plus the loader's 8-byte tail, with frame 0 all ones and frame 1 all zeros
so that every field takes its largest and smallest value.  Frame sizes are odd, so every track meets every `offset & 7` alignment.

At or past the end of a clip of 257 frames or more the sampler reads frame frame_count + 1 at t == 0 (`frame_count - 0.00001f` rounds
back to frame_count).  The reference reads past its stream there, and its result is defined only because t == 0; the library commits to
the clip's last frame.  `with_last_frame_repeated` gives both the restatement and the reference harness a copy of a clip whose streams
hold that frame once more, bit for bit, so that neither reads past its buffer.

Here the restatement is pinned to the reference's own code on those inputs (skipped where oracle/_ref was not built), with one exception:
the root-motion tables.  The reference keeps frame_count + 1 entries of pose_translations / pose_rotations and reads entry
frame_count + 1 past them at the end of a long clip; the restatement (oracle_stack_rm) repeats the last entry there, the value the library
commits to, and that entry has no reference value to be pinned to.  The root-motion pins below use the width clips, all shorter than 257
frames, whose reads stay inside the tables; the root-motion bone at the end of a long clip is held only to the restatement's choice."""
import ctypes as C
import os

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from lumixengine_b200.animation import CONST_R_DTYPE, CONST_T_DTYPE, TRACK_DTYPE, AnimationClip
from oracle import pyoracle as po
from oracle import pyrootmotion as prm
from oracle import pystack

from bitexact import assert_bits_equal

SHIM = po.ANIMATION_SHIM_SO
U32_MAX = 0xFFFFFFFF
BELOW = float(np.nextafter(np.float32(0.9999), np.float32(0)))

FRAME_COUNTS = (1, 2, 255, 256, 257, 300, 1000, 4097)
FPS = (1.0, 24.0, 25.0, 30.0, 59.94, 60.0)

# translation widths: channel 0 runs 1 .. 32, channels 1 and 2 run through 1 .. 32 in another order (7 and 13 are odd), then the wide ones
T_WIDTHS = [(w, (7 * w) % 32 + 1, (13 * w + 5) % 32 + 1) for w in range(1, 33)] + \
           [(32, 32, 32), (31, 31, 31), (33, 2, 9), (5, 47, 3), (1, 1, 63), (40, 40, 40), (63, 63, 63)]


def _rotation_widths():
    """Widths clampBitsizes lets through (each kept channel 1 .. 31, at most 48 together), every width 1 .. 31 in every channel, then
    slow-path ones: a 32-bit channel next to another, channels of 33 to 55 bits, and tracks wider than the 57 bits an 8-byte read keeps."""
    out = []
    for w in range(1, 32):
        a = (5 * w) % 16 + 1
        b = max(1, min((11 * w + 3) % 16 + 1, 48 - w - a))
        t = [w, a, b]
        k = w % 3
        out.append(tuple(t[k:] + t[:k]))
    return out + [(16, 16, 16), (31, 16, 1), (32, 1, 1), (32, 16, 1), (33, 10, 5), (2, 45, 3), (1, 1, 55), (20, 20, 20), (31, 31, 1)]


R_WIDTHS = _rotation_widths()


def _frame_bits(widths, extra):
    """Offsets of the tracks inside a frame and the frame size, made odd by one unused bit where the sum is even."""
    sizes = [sum(w) + extra for w in widths]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    total = int(sum(sizes))
    return offsets, total + (1 - total % 2)


def _stream(rng, frame_bits, frames):
    """Random stream of `frames` frames (+ the 8-byte tail) as bytes, frame 0 all ones, frame 1 all zeros."""
    n = (frame_bits * frames + 7) // 8
    big = int.from_bytes(rng.integers(0, 256, n + 8, dtype=np.uint8).tobytes(), "little")
    big |= (1 << frame_bits) - 1
    if frames > 1:
        big &= ~(((1 << frame_bits) - 1) << frame_bits)
    return np.frombuffer(big.to_bytes(n + 8, "little"), np.uint8).copy()


def raw_clip(sk, frames, fps, t_widths, r_widths, seed, t_bones=None, r_bones=None, n_const=2, negative_zero=False):
    """A clip of `frames` frames with one translation track per width set of t_widths (bones t_bones, default 0, 1, ...) and one rotation
    track per set of r_widths, over random stream bytes.  min / to_range keep translations within a few units and rotation channels
    within +-0.58, so that every quaternion is close to unit length.  n_const bones after the tracked ones get constant tracks."""
    rng = np.random.default_rng(seed)
    B = sk.bone_count
    t_bones = list(range(len(t_widths))) if t_bones is None else list(t_bones)
    r_bones = list(range(len(r_widths))) if r_bones is None else list(r_bones)
    assert len(set(t_bones)) == len(t_bones) <= B and len(set(r_bones)) == len(r_bones) <= B
    t_off, t_bits = _frame_bits(t_widths, 0)
    r_off, r_bits = _frame_bits(r_widths, 1)
    T = np.zeros(len(t_widths), TRACK_DTYPE)
    for i, (w, b) in enumerate(zip(t_widths, t_bones)):
        scale = np.array([float((1 << x) - 1) for x in w])
        mn = rng.uniform(-2.0, 2.0, 3)
        rng_ = rng.uniform(0.3, 3.0, 3) * rng.choice([-1.0, 1.0], 3) / scale
        if negative_zero or i % 7 == 3:
            mn[i % 3] = -0.0
        T[i] = (b, t_off[i], w, 0, mn.astype(np.float32), rng_.astype(np.float32))
    R = np.zeros(len(r_widths), TRACK_DTYPE)
    for i, (w, b) in enumerate(zip(r_widths, r_bones)):
        scale = np.array([float((1 << x) - 1) for x in w])
        mn = -0.57 + rng.uniform(-0.01, 0.01, 3)
        R[i] = (b, r_off[i], w, rng.integers(0, 4), mn.astype(np.float32), (1.14 / scale).astype(np.float32))
    free_t = [b for b in range(B) if b not in t_bones][:n_const]
    free_r = [b for b in range(B) if b not in r_bones][:n_const]
    CT = np.zeros(len(free_t), CONST_T_DTYPE)
    for i, b in enumerate(free_t):
        CT[i] = (b, 0, rng.normal(size=3).astype(np.float32))
    CR = np.zeros(len(free_r), CONST_R_DTYPE)
    for i, b in enumerate(free_r):
        q = rng.normal(size=4)
        CR[i] = (b, 0, (q / np.linalg.norm(q)).astype(np.float32))
    ts = _stream(rng, t_bits, frames + 1) if len(T) else np.zeros(8, np.uint8)
    rs = _stream(rng, r_bits, frames + 1) if len(R) else np.zeros(8, np.uint8)
    return AnimationClip(fps, frames, T, CT, R, CR, ts, rs, t_bits if len(T) else 0, r_bits if len(R) else 0)


def _repeat_last(stream, frame_bits, frame_count):
    if frame_bits == 0:
        return stream.copy()
    big = int.from_bytes(stream.tobytes(), "little")
    mask = (1 << frame_bits) - 1
    last = (big >> (frame_count * frame_bits)) & mask
    kept = big & ((1 << ((frame_count + 1) * frame_bits)) - 1)
    n = (frame_bits * (frame_count + 2) + 7) // 8 + 8
    return np.frombuffer((kept | (last << ((frame_count + 1) * frame_bits))).to_bytes(n, "little"), np.uint8).copy()


def with_last_frame_repeated(clip):
    """The same clip whose streams hold frame frame_count a second time as frame frame_count + 1 (same frame count, fps and tracks)."""
    return AnimationClip(clip.fps, clip.frame_count, clip.translations, clip.const_translations, clip.rotations, clip.const_rotations,
                         _repeat_last(clip.translation_stream, clip.translations_frame_size_bits, clip.frame_count),
                         _repeat_last(clip.rotation_stream, clip.rotations_frame_size_bits, clip.frame_count),
                         clip.translations_frame_size_bits, clip.rotations_frame_size_bits, clip.flags)


def end_times(clip):
    L = clip.length_ticks
    return [0, L - 1, L, L + 1, L + 4000, U32_MAX]


def length_inputs():
    """(skeleton, clips): every frame count at every fps, the tracks on the root (bone 0, the root-motion bone) and below it, widths
    taken in turn from the sets of T_WIDTHS / R_WIDTHS whose tracks fit in 57 bits.  A wider track loses the bits past the 8 bytes it
    is read from, and which ones depends on the frame's alignment: the repeated frame would not decode to the last frame's values."""
    sk = scenes.skeleton(seed=6, parents=[-1, 0, 1, 1, 3, 0])
    t_narrow = [w for w in T_WIDTHS if sum(w) <= 57]
    r_narrow = [w for w in R_WIDTHS if sum(w) + 1 <= 57]
    clips = []
    for i, fc in enumerate(FRAME_COUNTS):
        for j, fps in enumerate(FPS):
            k = len(clips)
            tw = [t_narrow[(k + m) % len(t_narrow)] for m in range(3)]
            rw = [r_narrow[(k + m) % len(r_narrow)] for m in range(3)]
            clips.append(raw_clip(sk, fc, fps, tw, rw, seed=1000 + k, t_bones=(0, 2, 4), r_bones=(0, 3, 5)))
    return sk, clips


def width_inputs():
    """(skeleton, clips): clip j gives track m the width set (m + j) % n, so the root-motion bone 0 (track 0) meets every width set in
    some clip and every clip holds every width set.  9 to 48 frames, several fps."""
    sk = scenes.skeleton(64, seed=8)
    clips = []
    for j in range(len(T_WIDTHS)):
        tw = [T_WIDTHS[(m + j) % len(T_WIDTHS)] for m in range(len(T_WIDTHS))]
        rw = [R_WIDTHS[(m + j) % len(R_WIDTHS)] for m in range(len(R_WIDTHS))]
        perm = np.random.default_rng(j).permutation(np.arange(1, sk.bone_count))
        t_bones = [0] + [int(b) for b in perm[:len(tw) - 1]]
        r_bones = [0] + [int(b) for b in perm[::-1][:len(rw) - 1]]
        clips.append(raw_clip(sk, 9 + (7 * j) % 40, FPS[j % len(FPS)], tw, rw, seed=2000 + j, t_bones=t_bones, r_bones=r_bones))
    return sk, clips


LENGTHS = length_inputs()
WIDTHS = width_inputs()


def test_inputs_cover_the_edges():
    for sk, clips in (LENGTHS, WIDTHS):
        for c in clips:
            for tracks, bits, stream in ((c.translations, c.translations_frame_size_bits, c.translation_stream),
                                         (c.rotations, c.rotations_frame_size_bits, c.rotation_stream)):
                assert len(stream) == (bits * (c.frame_count + 1) + 7) // 8 + 8  # exactly what lb200_animation_create takes
                assert bits % 2 == 1
                if c.frame_count >= 8:  # an odd frame size walks a track through every alignment
                    for off in tracks["offset_bits"]:
                        assert {(bits * f + int(off)) & 7 for f in range(8)} == set(range(8))
    t = np.concatenate([c.translations["bitsizes"] for c in WIDTHS[1]])
    for ch in range(3):
        assert set(range(1, 33)) <= set(t[:, ch].tolist()), ch
    assert {33, 40, 47, 63} <= set(t.ravel().tolist())
    r = np.concatenate([c.rotations["bitsizes"] for c in WIDTHS[1]])
    assert set(range(1, 33)) <= set(r.ravel().tolist()) and all(r[:, ch].max() >= 31 for ch in range(3))
    assert max(int(x.sum()) for x in r) + 1 > 57 and max(int(x.sum()) for x in t) > 57
    assert {c.frame_count for c in LENGTHS[1]} == set(FRAME_COUNTS) and {np.float32(c.fps) for c in LENGTHS[1]} == {np.float32(f) for f in FPS}


def test_the_repeated_frame_is_the_last_one():
    """with_last_frame_repeated changes nothing before the end: frames 0 .. frame_count decode to the same bytes, and frame frame_count + 1
    to those of frame frame_count."""
    sk, clips = LENGTHS
    for c in clips[::5]:
        e = with_last_frame_repeated(c)
        f = np.arange(c.frame_count + 1, dtype=np.uint32)
        for r in range(len(c.rotations)):
            assert_bits_equal(prm.rotation_d(e, r, f), prm.rotation_d(c, r, f), "rotations before the end")
            assert_bits_equal(prm.rotation_d(e, r, [c.frame_count + 1]), prm.rotation_d(c, r, [c.frame_count]), "the repeated frame")
        inside = [0, c.length_ticks // 3, c.length_ticks - 1]
        for t in inside:
            a, b = po.pose_evaluate(sk, e, t), po.pose_evaluate(sk, c, t)
            assert_bits_equal(a[0], b[0], "positions inside the clip")
            assert_bits_equal(a[1], b[1], "rotations inside the clip")


def test_long_clip_ends_reach_the_repeated_frame():
    """The inputs are not vacuous: for the clips of 257 frames or more, some end time samples frame frame_count itself."""
    sk, clips = LENGTHS
    hit = set()
    for c in clips:
        hi = np.float32(np.float32(c.frame_count) - np.float32(0.00001))
        for t in end_times(c)[2:]:
            frame = np.float32(t / 32768.0 * np.float64(np.float32(c.fps)))
            if min(max(frame, np.float32(0)), hi) >= c.frame_count:
                hit.add(c.frame_count)
    assert hit == {fc for fc in FRAME_COUNTS if fc >= 257}


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.ref_available():
        pytest.skip("oracle/_ref/libref_lumix.so not built (needs the reference tree)")
    return oracle


def _pin(a, b, what):
    assert_bits_equal(a[0], b[0], f"{what}: positions")
    assert_bits_equal(a[1], b[1], f"{what}: rotations")


def test_widths_equal_reference(ref):
    """Animation::getRelativePose (+ Pose::computeAbsolute) at every width, plain and weighted on top of another sample."""
    sk, clips = WIDTHS
    rng = np.random.default_rng(5)
    for j, c in enumerate(clips):
        e = with_last_frame_repeated(c)
        for t in end_times(c) + [int(x) for x in rng.integers(0, c.length_ticks, 3)]:
            for absolute in (False, True):
                _pin(ref.pose_evaluate(sk, e, t, compute_absolute=absolute), ref.ref_pose_evaluate(sk, e, t, compute_absolute=absolute), f"clip {j} t={t}")
            base = ref.pose_evaluate(sk, clips[(j + 1) % len(clips)], 0, compute_absolute=False)
            for w in (0.5, BELOW):
                kw = dict(weight=w, start_from_bind=False, compute_absolute=True, pos=base[0], rot=base[1])
                _pin(ref.pose_evaluate(sk, e, t, **kw), ref.ref_pose_evaluate(sk, e, t, **kw), f"clip {j} t={t} w={w}")


def test_long_clip_ends_equal_reference(ref):
    sk, clips = LENGTHS
    for j, c in enumerate(clips):
        e = with_last_frame_repeated(c)
        for t in end_times(c):
            _pin(ref.pose_evaluate(sk, e, t), ref.ref_pose_evaluate(sk, e, t), f"{c.frame_count} frames at {c.fps} fps, t={t}")


def _shim():
    if not os.path.exists(SHIM):
        pytest.skip("root-motion harness not built (no reference tree where build() ran)")
    return C.CDLL(SHIM)


def _ref_stack(L, sk, clips, ci, t, w, lo):
    B = sk.bone_count
    pos, rot = np.zeros((B, 3), np.float32), np.zeros((B, 4), np.float32)
    arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    P = po._ptr
    assert L.ref_pose_stack(C.byref(po._skeleton_struct(sk, po.RefSkeleton)), arr, C.c_uint32(len(clips)), P(np.ascontiguousarray(ci, np.uint32)),
                            P(np.ascontiguousarray(w, np.float32)), P(np.ascontiguousarray(t, np.uint32)), P(np.ascontiguousarray(lo, np.uint32)),
                            C.c_uint32(len(ci)), P(pos), P(rot)) == 0
    return pos, rot


def stack_plan(clips, n, seed):
    """n samples over `clips`: end times, looped and clamped, weights on both sides of 0.9999."""
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    t = np.array([end_times(clips[c])[k] for c, k in zip(ci, rng.integers(0, 6, n))], np.uint32)
    w = rng.choice(np.array([1.0, 0.99995, 0.9999, BELOW, 0.5], np.float32), n)
    lo = rng.integers(0, 2, n).astype(np.uint32)
    return ci, t, w, lo


def test_stacks_equal_reference():
    """getPose + evalBlendStack: looped and clamped samples at the clip ends, on both input sets."""
    L = _shim()
    for name, (sk, clips) in (("lengths", LENGTHS), ("widths", WIDTHS)):
        ext = [with_last_frame_repeated(c) for c in clips]
        for k in range(12):
            ci, t, w, lo = stack_plan(clips, 1 + k % 3, seed=k)
            _pin(pystack.pose_stack(sk, ext, ci, t, w, lo), _ref_stack(L, sk, ext, ci, t, w, lo), f"{name} stack {k}")


def test_root_motion_widths_equal_reference():
    """setRootMotionBone's tables, Animation::getRotation through fp64 and the sampling of the tables, with the root-motion bone's
    tracks at every width set."""
    from test_animation_root_motion_cpu import run_ref_math, run_ref_pose_stack, run_ref_tables
    L = _shim()
    sk, clips = WIDTHS
    tt, rt = np.zeros(len(clips), np.int32), np.zeros(len(clips), np.int32)  # track 0 of every clip is bone 0's
    for j, c in enumerate(clips):
        assert c.rootMotionTracks(0) == (0, 0)
        flags = 1 + j % 7
        t, r, pt, pr = run_ref_tables(L, c, flags, 0)
        ok, ept, epr = prm.tables(c, flags, 0, 0)
        assert ok and (t, r) == (0, 0)
        assert_bits_equal(ept, pt, f"clip {j}: pose_translations")
        assert_bits_equal(epr, pr, f"clip {j}: pose_rotations")
        for track in range(0, len(c.rotations), 9):
            _, rot = run_ref_math(L, np.zeros((1, 4), np.float32), c, track)
            assert_bits_equal(prm.rotation_d(c, track, np.arange(c.frame_count + 1)), rot, f"clip {j}: getRotation of track {track}")
    flags = np.array([1 + j % 7 for j in range(len(clips))], np.uint32)
    rm = prm.root_motion(flags, tt, rt)
    for k in range(12):
        ci, t, w, lo = stack_plan(clips, 1 + k % 3, seed=100 + k)  # clips under 257 frames: every read stays inside the tables
        _pin(prm.pose_stack(sk, clips, rm, ci, t, w, lo), run_ref_pose_stack(L, sk, clips, flags, 0, ci, t, w, lo), f"root-motion stack {k}")
