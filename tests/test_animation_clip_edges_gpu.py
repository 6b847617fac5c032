"""The pose kernels on long clips at and past their end and on every channel width, bit for bit against the restatement.

The inputs are tests/test_animation_clip_edges_cpu.py's (pinned there to the reference's own code): LENGTHS, 48 clips of 1 to 4097
frames at 1 to 60 fps, every one sampled at 0, L - 1, L, L + 1, L + 4000 and 2^32 - 1 ticks; WIDTHS, 39 clips of raw bit streams with
channels of 1 to 63 bits.  Every pose mode runs on them: clip mode, clip mode with two layers (weights below and above 0.9999), sample lists
(looped and clamped), stacks with one IK op and sample lists over clips with root motion, at every lane count and through update_many; the
long clips run once with each of them last in its system.  Absolute poses, dual quaternions, matrices and advanced times must equal the
restatement's.  The restatement samples the clips with their last frame repeated (with_last_frame_repeated), which is what the library
commits to where the sampler reads past the last frame.

Then a clip whose last frame decodes to -0.0, in a translation and in a rotation channel, in front of a clip whose first row would turn
both into +0.0, and the refusals of lb200_animation_create with the largest clips it accepts."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from lumixengine_b200.animation import CONST_R_DTYPE, CONST_T_DTYPE, TRACK_DTYPE, AnimationClip, _pack_frames
from oracle import pyoracle as po
from oracle import pyrootmotion as prm
from oracle import pystack
from bitexact import assert_bits_equal
from test_animation_clip_edges_cpu import BELOW, FPS, FRAME_COUNTS, LENGTHS, U32_MAX, WIDTHS, end_times, raw_clip, stack_plan, with_last_frame_repeated

pytestmark = pytest.mark.gpu

ALL = lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE
ERR_INVALID = lb._lib.ERR_INVALID
MODES = ("clips", "layers", "lists", "ik", "root_motion")
INPUTS = {"lengths": LENGTHS, "widths": WIDTHS}
STEP = {4: 1.0 / 30.0, 8: -0.37, 16: 0.0, 32: 2.5}  # time step per lane count: > 0, < 0 and 0


def _deepest(sk):
    depth = np.zeros(sk.bone_count, np.int64)
    for b in range(sk.bone_count):
        depth[b] = 0 if sk.parents[b] < 0 else depth[sk.parents[b]] + 1
    leaf = int(np.argmax(depth))
    return leaf, int(depth[leaf]) + 1


_PLANS = {}


def plan(name, mode):
    """The instances of one mode over canonical clip indices."""
    key = (name, mode)
    if key in _PLANS:
        return _PLANS[key]
    sk, clips = INPUTS[name]
    seed = 10 * list(INPUTS).index(name) + MODES.index(mode)
    rng = np.random.default_rng(seed)
    nc = len(clips)
    if mode in ("clips", "layers"):
        ci, t = [], []
        for c in range(nc):
            times = end_times(clips[c]) + [int(x) for x in rng.integers(0, clips[c].length_ticks, 2)]
            ci += [c] * len(times)
            t += times
        ci, t = np.array(ci, np.uint32), np.array(t, np.uint32)
        n = len(ci)
        L = 2 if mode == "layers" else 0
        lc = rng.integers(0, nc, (n, L)).astype(np.uint32)
        lt = np.array([[end_times(clips[c])[k] for c, k in zip(row, rng.integers(0, 6, L))] for row in lc], np.uint32).reshape(n, L)
        lw = np.zeros((n, L), np.float32)
        if L:
            lw[:, 0] = rng.choice(np.array([0.5, BELOW, 0.25], np.float32), n)
            lw[:, 1] = rng.choice(np.array([1.0, 0.99995, 0.9999], np.float32), n)
        p = dict(ci=ci, t=t, lc=lc, lt=lt, lw=lw, n=n)
    else:
        n = 160
        counts = rng.integers(1, 4, n)
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
        ci, t, w, lo = stack_plan(clips, int(offsets[-1]), seed=seed + 50)
        p = dict(offsets=offsets, ci=ci, t=t, w=w, lo=lo, n=n)
        if mode == "ik":
            leaf, path = _deepest(sk)
            p.update(ik_offsets=np.arange(n + 1, dtype=np.uint32), after=np.array([rng.integers(0, c + 1) for c in counts], np.uint32),
                     leaf=np.full(n, leaf, np.uint32), bones=rng.integers(2, min(path, 3) + 1, n).astype(np.uint32),
                     alpha=rng.choice(np.array([1.0, 0.7], np.float32), n), target=(rng.normal(size=(n, 3)) * 0.5).astype(np.float32))
        if mode == "root_motion":
            tr = np.array([c.rootMotionTracks(0) for c in clips], np.int32)
            p.update(rm=prm.root_motion(1 + np.arange(nc) % 7, tr[:, 0], tr[:, 1]))
    _PLANS[key] = p
    return p


_EXPECTED = {}


def expected(name, mode):
    key = (name, mode)
    if key in _EXPECTED:
        return _EXPECTED[key]
    sk, clips = INPUTS[name]
    ext = [with_last_frame_repeated(c) for c in clips]
    p = plan(name, mode)
    n, B = p["n"], sk.bone_count
    if mode == "clips":
        out = po.animate_instances(sk, ext, p["ci"], p["t"])
    else:
        out = dict(pos=np.empty((n, B, 3), np.float32), rot=np.empty((n, B, 4), np.float32), dq=np.empty((n, B, 8), np.float32), mtx=np.empty((n, B, 16), np.float32))
        for i in range(n):
            if mode == "layers":
                pr = po.pose_evaluate(sk, ext[p["ci"][i]], p["t"][i], compute_absolute=False)
                for k in range(p["lc"].shape[1]):
                    pr = po.pose_evaluate(sk, ext[p["lc"][i, k]], p["lt"][i, k], weight=float(p["lw"][i, k]), start_from_bind=False, compute_absolute=False,
                                          pos=pr[0], rot=pr[1])
                pr = po.pose_compute_absolute(sk, *pr)
            else:
                s = slice(p["offsets"][i], p["offsets"][i + 1])
                args = (p["ci"][s], p["t"][s], p["w"][s], p["lo"][s])
                if mode == "lists":
                    pr = pystack.pose_stack(sk, ext, *args)
                elif mode == "ik":
                    pr = prm.pose_stack(sk, ext, None, *args, p["after"][i:i + 1], p["leaf"][i:i + 1], p["bones"][i:i + 1], p["alpha"][i:i + 1], p["target"][i:i + 1])
                else:
                    pr = prm.pose_stack(sk, ext, p["rm"], *args)
            out["pos"][i], out["rot"][i] = pr
            out["dq"][i], out["mtx"][i] = po.palettes(sk, *pr)
    _EXPECTED[key] = out
    return out


def _system(ctx, name, mode, order, G=0):
    """The mode's instances on a system whose clips are the inputs' in `order` (canonical indices)."""
    sk, clips = INPUTS[name]
    p = plan(name, mode)
    at = np.empty(len(order), np.uint32)
    at[np.asarray(order)] = np.arange(len(order))  # canonical index -> index in the system
    a = lb.AnimationSystem(ctx, sk, [clips[c] for c in order], None, max_instances=p["n"])
    a.setLaunch(G, 0)
    if mode in ("clips", "layers"):
        a.setInstances(at[p["ci"]], p["t"])
        if mode == "layers":
            a.setLayers(at[p["lc"]], p["lt"], p["lw"])
    elif mode == "ik":
        a.setStacks(p["offsets"], at[p["ci"]], p["t"], p["w"], p["lo"], p["ik_offsets"], p["after"], p["leaf"], p["bones"], p["alpha"], p["target"])
    else:
        a.setSamples(p["offsets"], at[p["ci"]], p["t"], p["w"], p["lo"])
        if mode == "root_motion":
            rm = p["rm"][np.asarray(order)]
            a.setRootMotion(rm["flags"], rm["translation_track"], rm["rotation_track"])
    return a


def _check(a, name, mode, dt, what):
    exp = expected(name, mode)
    p, r = a.getPose()
    assert_bits_equal(p, exp["pos"], f"{what}: pose.pos")
    assert_bits_equal(r, exp["rot"], f"{what}: pose.rot")
    assert_bits_equal(a.getDualQuats(), exp["dq"], f"{what}: dual quats")
    assert_bits_equal(a.getMatrices(), exp["mtx"], f"{what}: matrices")
    if mode in ("clips", "layers"):
        clips = INPUTS[name][1]
        pl = plan(name, mode)
        want = np.array([po.time_advance(t, dt, clips[c].fps, clips[c].frame_count) for c, t in zip(pl["ci"], pl["t"])], np.uint32)
        assert_bits_equal(a.getTimes(), want, f"{what}: advanced times")


def _last_orders():
    """One clip order per long frame count, that count's clip (at one of the frame rates in turn) last; the canonical order ends with the
    4097-frame clip at 60 fps."""
    clips = LENGTHS[1]
    orders = {}
    for k, fc in enumerate(fc for fc in FRAME_COUNTS if fc >= 255):
        last = next(i for i, c in enumerate(clips) if c.frame_count == fc and np.float32(c.fps) == np.float32(FPS[k % len(FPS)]))
        orders[fc] = [i for i in range(len(clips)) if i != last] + [last]
    return orders


LAST_ORDERS = _last_orders()


@pytest.mark.parametrize("G", [4, 8, 16, 32])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(INPUTS))
def test_every_mode_every_lane_count(ctx, name, mode, G):
    a = _system(ctx, name, mode, list(range(len(INPUTS[name][1]))), G)
    a.update(STEP[G], ALL)
    assert a.lastLaunch()[0] == G
    _check(a, name, mode, STEP[G], f"{name} {mode} G={G}")
    a.close()


@pytest.mark.parametrize("last", list(LAST_ORDERS))
@pytest.mark.parametrize("mode", MODES)
def test_each_long_clip_last_in_its_system(ctx, mode, last):
    a = _system(ctx, "lengths", mode, LAST_ORDERS[last])
    a.update(1.0 / 60.0, ALL)
    _check(a, "lengths", mode, 1.0 / 60.0, f"{mode}, the {last}-frame clip last")
    a.close()


@pytest.mark.parametrize("mode", MODES)
def test_update_many(ctx, mode):
    """Every clip order of the long clips and the width clips in one update_many."""
    runs = [("lengths", o) for o in LAST_ORDERS.values()] + [("widths", list(range(len(WIDTHS[1]))))]
    systems = [_system(ctx, name, mode, order) for name, order in runs]
    lb.AnimationSystem.updateMany(systems, -1.0 / 30.0, ALL)
    for k, ((name, _), a) in enumerate(zip(runs, systems)):
        _check(a, name, mode, -1.0 / 30.0, f"{mode}: system {k} of update_many ({name})")
        a.close()


def _bone0_clip(frames, fps, t_fields, t_min, t_range, r_fields=None, r_min=None, r_range=None, const_rot=(0.0, 0.0, 0.0, 1.0)):
    """A clip with one 8-8-8-bit translation track on bone 0 (fields t_fields [frames + 1, 3]) and either one 8-8-8-bit rotation track on
    bone 0 (fields r_fields, sign bit 0, w the skipped channel) or the constant rotation const_rot."""
    v = np.asarray(t_fields, np.uint64)
    stream, offsets, bits = _pack_frames([v[:, 0] | (v[:, 1] << np.uint64(8)) | (v[:, 2] << np.uint64(16))], [24])
    T = np.zeros(1, TRACK_DTYPE)
    T[0] = (0, offsets[0], (8, 8, 8), 0, t_min, t_range)
    R, CR = np.zeros(0, TRACK_DTYPE), np.zeros(0, CONST_R_DTYPE)
    r_stream, r_bits = np.zeros(8, np.uint8), 0
    if r_fields is None:
        CR = np.zeros(1, CONST_R_DTYPE)
        CR[0] = (0, 0, const_rot)
    else:
        v = np.asarray(r_fields, np.uint64)
        r_stream, r_off, r_bits = _pack_frames([(v[:, 0] | (v[:, 1] << np.uint64(8)) | (v[:, 2] << np.uint64(16))) << np.uint64(1)], [25])
        R = np.zeros(1, TRACK_DTYPE)
        R[0] = (0, r_off[0], (8, 8, 8), 3, r_min, r_range)
    return AnimationClip(fps, frames, T, np.zeros(0, CONST_T_DTYPE), R, CR, stream, r_stream, bits, r_bits)


def _negative_zero(x):
    return np.all(x == 0) and np.all(np.signbit(x))


def test_negative_zero_at_the_end(ctx):
    """A 300-frame clip whose last frame decodes to -0.0 in a translation channel (min -0.0, a negative to_range, field 0) and in a rotation
    channel (the same, the quaternion (-0.0, 0.6, 0, 0.8)), followed by a clip whose row 0 holds 1.0 and a rotation of negative x and
    negative dot with that quaternion.  At the clip's end the sampler mixes the last frame with the row after it at t == 0:
      lerp: -0.0 * 1 + x * 0 keeps the sign only when x is -0.0 too, the last frame again; the next clip's 1.0 gives +0.0;
      simd_nlerp: a negative dot turns t into -0.0, and -0.0 * 1 + (-0.6) * -0.0 is +0.0; the last frame again keeps -0.0.
    So only the repeated last frame gives the reference's -0.0 in both."""
    sk = scenes.skeleton(seed=3, parents=[-1, 0])
    rng = np.random.default_rng(1)
    t_fields = rng.integers(1, 256, (301, 3))
    t_fields[300] = 0
    r_fields = rng.integers(1, 256, (301, 3))
    r_fields[300] = 0
    a_clip = _bone0_clip(300, 30.0, t_fields, np.full(3, -0.0, np.float32), np.full(3, -0.01, np.float32),
                         r_fields, np.array([-0.0, 0.6, 0.0], np.float32), np.array([-0.001, 0.001, 0.001], np.float32))
    q2 = np.array([-0.6, -0.6, 0.0, -0.53], np.float64)
    b_clip = _bone0_clip(10, 30.0, rng.integers(0, 256, (11, 3)), np.ones(3, np.float32), np.full(3, 0.01, np.float32),
                         const_rot=tuple((q2 / np.linalg.norm(q2)).astype(np.float32)))
    clips = [a_clip, b_clip]
    L = a_clip.length_ticks
    times = np.array([L, L + 1, L + 4000, U32_MAX], np.uint32)
    ext = [with_last_frame_repeated(c) for c in clips]
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=8)
    for G in (4, 8, 16, 32):
        a.setLaunch(G, 0)
        a.setInstances(np.zeros(len(times), np.uint32), times)
        a.update(0.0, ALL)
        pos, rot = a.getPose()
        assert _negative_zero(pos[:, 0]), f"G={G}: bone 0's position at the clip's end is {pos[:, 0]}, not -0.0"
        assert _negative_zero(rot[:, 0, 0]), f"G={G}: bone 0's rotation x at the clip's end is {rot[:, 0, 0]}, not -0.0"
        exp = po.animate_instances(sk, ext, np.zeros(len(times), np.uint32), times)
        assert_bits_equal(pos, exp["pos"], f"G={G}: clip mode positions")
        assert_bits_equal(rot, exp["rot"], f"G={G}: clip mode rotations")
        assert_bits_equal(a.getDualQuats(), exp["dq"], f"G={G}: clip mode dual quats")
        # the same end as a clamped sample-list entry (getPose sets it to exactly the length) and as a layer
        a.setSamples(np.arange(len(times) + 1, dtype=np.uint32), np.zeros(len(times)), times, np.ones(len(times)), np.zeros(len(times)))
        a.update(0.0, ALL)
        pos, rot = a.getPose()
        assert _negative_zero(pos[:, 0]) and _negative_zero(rot[:, 0, 0]), f"G={G}: clamped samples"
        for i, t in enumerate(times):
            want = pystack.pose_stack(sk, ext, [0], [t], [1.0], [0])
            assert_bits_equal(pos[i], want[0], f"G={G}: clamped sample at {t}: positions")
            assert_bits_equal(rot[i], want[1], f"G={G}: clamped sample at {t}: rotations")
        a.setInstances(np.ones(len(times), np.uint32), np.zeros(len(times), np.uint32))
        a.setLayers(np.zeros((len(times), 1)), times[:, None], np.ones((len(times), 1)))
        a.update(0.0, ALL)
        pos, rot = a.getPose()
        assert _negative_zero(pos[:, 0]) and _negative_zero(rot[:, 0, 0]), f"G={G}: layers"
    a.close()


def _const_clip(frames, fps, t_bone=0, r_bone=None):
    CT = np.zeros(1, CONST_T_DTYPE)
    CT[0] = (t_bone, 0, (0.5, 0.25, 0.0))
    CR = np.zeros(0 if r_bone is None else 1, CONST_R_DTYPE)
    if r_bone is not None:
        CR[0] = (r_bone, 0, (0.0, 0.0, 0.0, 1.0))
    return AnimationClip(fps, frames, np.zeros(0, TRACK_DTYPE), CT, np.zeros(0, TRACK_DTYPE), CR, np.zeros(8, np.uint8), np.zeros(8, np.uint8), 0, 0)


def _with_bits(clip, kind, track, channel, bits):
    c = AnimationClip(clip.fps, clip.frame_count, clip.translations.copy(), clip.const_translations, clip.rotations.copy(), clip.const_rotations,
                      clip.translation_stream, clip.rotation_stream, clip.translations_frame_size_bits, clip.rotations_frame_size_bits)
    getattr(c, kind)[track]["bitsizes"][channel] = bits
    return c


def test_create_refusals(ctx):
    """lb200_animation_create refuses, with LB200_ERR_INVALID and before it allocates, what the reference leaves undefined or the tables
    cannot address; the context keeps working after every refusal."""
    sk = scenes.skeleton(seed=2, parents=[-1, 0])
    sk196 = scenes.skeleton(196)
    ok = WIDTHS[1][0]
    wide_sk = WIDTHS[0]
    refused = {
        "no frames": (sk, [_const_clip(0, 30.0)]),
        "fps 0": (sk, [_const_clip(10, 0.0)]),
        "fps < 0": (sk, [_const_clip(10, -30.0)]),
        "fps NaN": (sk, [_const_clip(10, float("nan"))]),
        "shorter than one tick": (sk, [_const_clip(1, 1.0e6)]),
        "2^32 ticks": (sk, [_const_clip(131072, 1.0)]),
        "far past 2^32 ticks": (sk, [_const_clip(0xFFFFFFFF, 30.0)]),
        "a 64-bit translation channel": (wide_sk, [_with_bits(ok, "translations", 3, 0, 64)]),
        "a 255-bit translation channel": (wide_sk, [_with_bits(ok, "translations", 0, 2, 255)]),
        "a 64-bit rotation channel": (wide_sk, [_with_bits(ok, "rotations", 5, 1, 64)]),
        "a constant translation of bone 2 on 2 bones": (sk, [_const_clip(10, 30.0, t_bone=2)]),
        "a constant rotation of bone 2 on 2 bones": (sk, [_const_clip(10, 30.0, r_bone=2)]),
        # from 2^24 frames the fp32 clamp frame_count - 0.00001f can round above frame_count (2^24 + 3 rounds to 2^24 + 4)
        "2^24 frames": (sk, [_const_clip(1 << 24, 256.0)]),
        "2^24 + 3 frames": (sk, [_const_clip((1 << 24) + 3, 256.0)]),
        "2^32 - 1 frames": (sk, [_const_clip(0xFFFFFFFF, 1.0e6)]),
        # 196 bones are 196 entries per row: (frame_count + 2) * 196 passes 2^31 - 1 while (frame_count + 1) * 196 does not
        "the repeated row past 2^31 entries": (sk196, [_const_clip(10956548, 128.0)]),
        "two clips past 2^31 entries": (sk196, [_const_clip(5478274, 128.0)] * 2),
    }
    for what, (s, clips) in refused.items():
        with pytest.raises(lb.LumixB200Error) as e:
            lb.AnimationSystem(ctx, s, clips, None, max_instances=1)
        assert e.value.code == ERR_INVALID, what
    # just inside: 63-bit channels (WIDTHS), a length one frame short of 2^32 ticks, and 2^24 - 1 frames with animated tracks, whose end
    # samples the repeated last row (frame_count - 0.00001f rounds to frame_count there)
    longest = raw_clip(sk, (1 << 24) - 1, 256.0, [(1, 1, 1)], [(1, 1, 1)], seed=9, t_bones=(0,), r_bones=(0,), n_const=1)
    for s, clips in ((sk, [_const_clip(131071, 1.0)]), (wide_sk, [_with_bits(ok, "translations", 3, 0, 63)]), (sk, [longest])):
        L = clips[0].length_ticks
        times = np.array([0, L - 1, L, L + 1, U32_MAX], np.uint32)
        a = lb.AnimationSystem(ctx, s, clips, None, max_instances=len(times))
        a.setInstances(np.zeros(len(times), np.uint32), times)
        a.update(0.0, ALL)
        exp = po.animate_instances(s, [with_last_frame_repeated(c) for c in clips], np.zeros(len(times), np.uint32), times)
        pos, rot = a.getPose()
        assert_bits_equal(pos, exp["pos"], f"accepted {clips[0].frame_count}-frame clip: positions")
        assert_bits_equal(rot, exp["rot"], f"accepted {clips[0].frame_count}-frame clip: rotations")
        a.close()
