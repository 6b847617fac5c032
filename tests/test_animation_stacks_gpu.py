"""lb200_animation_set_samples (AnimationSystem.setSamples): the SAMPLE instructions of animators' blend stacks posed on the device.

Every case is held bit for bit to oracle_pose_stack (the bind pose, getPose's time rule and Animation::getRelativePose per sample, then
computeAbsolute): absolute poses, dual quaternions and matrices.  The lists mix lengths 0 .. 40 per instance so that instances sharing a
warp differ, start below weight 0.9999, hit the weight edges (0, the float below 0.9999, 0.9999, 1, 2) and the time edges of looped and
clamped samples (0, length - 1, length, above length), over clips with constant, animated and untracked bones, at every lane count and on
1-, 64- and 196-bone skeletons.  Then: a list [base clip at weight 1, layers...] against clip mode + set_layers, update_many over both
modes against per-system updates, the pose consumers on a sample-list system, and the refusals.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from lumixengine_b200.animation import AnimationClip
from oracle import pyoracle as po
from oracle import pystack
from bitexact import assert_bits_equal

pytestmark = pytest.mark.gpu

DQ, MTX, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_MATRIX, lb.PALETTE_POSE
ALL = DQ | MTX | POSE
ERR_INVALID = lb._lib.ERR_INVALID
BELOW = float(np.nextafter(np.float32(0.9999), np.float32(0)))  # the float just below 0.9999f
WEIGHTS = [0.0, BELOW, 0.9999, 1.0, 2.0, 0.25, 0.5, 0.75]


@pytest.fixture(scope="module")
def ctx():
    c = lb.Context(0)
    yield c
    c.close()


def _partial(clip, keep):
    """The same clip with only the tracks of bones where keep[bone]: the other bones are untracked (they keep the pose below)."""
    f = lambda tracks: tracks[keep[tracks["bone_index"]]]  # noqa: E731
    return AnimationClip(clip.fps, clip.frame_count, f(clip.translations), f(clip.const_translations), f(clip.rotations), f(clip.const_rotations),
                         clip.translation_stream, clip.rotation_stream, clip.translations_frame_size_bits, clip.rotations_frame_size_bits)


def _setup(B, seed=3):
    sk = scenes.skeleton(64, seed=4) if B == 64 else scenes.skeleton(seed=B, parents=[-1] + [max(0, i - 1 - (i % 3)) for i in range(1, B)])
    rng = np.random.default_rng(seed)
    full = [scenes.clip(sk, frames=13, fps=30.0, seed=seed, const_fraction=0.3),
            scenes.clip(sk, frames=40, fps=24.0, seed=seed + 1, pos_bits=(11, 14, 16), rot_bits=(12, 15, 16), const_fraction=0.3)]
    keep = rng.random(B) < 0.5
    keep[0] = True
    clips = full + [_partial(full[0], keep), _partial(full[1], ~keep), scenes.clip(sk, frames=1, fps=60.0, seed=seed + 2, const_fraction=1.0)]
    return sk, clips


def _lists(n, clips, seed, lengths=(0, 1, 2, 3, 40)):
    """Per instance a list of random length from `lengths` (cycled over the first instances, so every length occurs), with the weight and
    time edges spread over the samples."""
    rng = np.random.default_rng(seed)
    counts = np.array([lengths[i % len(lengths)] if i < 2 * len(lengths) else lengths[rng.integers(0, len(lengths))] for i in range(n)], np.int64)
    rng.shuffle(counts[2 * len(lengths):])
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    total = int(offsets[-1])
    clip = rng.integers(0, len(clips), total).astype(np.uint32)
    L = np.array([c.length_ticks for c in clips], np.int64)[clip]
    edge = rng.integers(0, 6, total)
    t = np.where(edge == 0, 0, np.where(edge == 1, L - 1, np.where(edge == 2, L, np.where(edge == 3, L + 1 + rng.integers(0, 3 * L + 1),
                 (rng.random(total) * L).astype(np.int64)))))
    time_ticks = np.minimum(t, 0xFFFFFFFF).astype(np.uint32)
    weight = np.array(WEIGHTS, np.float32)[rng.integers(0, len(WEIGHTS), total)]
    looped = rng.integers(0, 2, total).astype(np.uint32)
    # every list of length >= 1 whose index is odd starts below 0.9999: its first sample blends towards the bind pose
    for i in range(1, n, 2):
        if counts[i]:
            weight[offsets[i]] = 0.5
    return offsets, clip, time_ticks, weight, looped


def _expected(sk, clips, offsets, clip, time_ticks, weight, looped):
    n, B = len(offsets) - 1, sk.bone_count
    pos = np.empty((n, B, 3), np.float32)
    rot = np.empty((n, B, 4), np.float32)
    dq = np.empty((n, B, 8), np.float32)
    mtx = np.empty((n, B, 16), np.float32)
    for i in range(n):
        a, b = int(offsets[i]), int(offsets[i + 1])
        pos[i], rot[i] = pystack.pose_stack(sk, clips, clip[a:b], time_ticks[a:b], weight[a:b], looped[a:b])
        dq[i], mtx[i] = po.palettes(sk, pos[i], rot[i])
    return dict(pos=pos, rot=rot, dq=dq, mtx=mtx)


def _check(anim, exp, what):
    p, r = anim.getPose()
    assert_bits_equal(p, exp["pos"], f"{what}: pose positions")
    assert_bits_equal(r, exp["rot"], f"{what}: pose rotations")
    assert_bits_equal(anim.getDualQuats(), exp["dq"], f"{what}: dual quaternions")
    assert_bits_equal(anim.getMatrices(), exp["mtx"], f"{what}: matrices")


@pytest.mark.parametrize("B", [1, 64, 196])
@pytest.mark.parametrize("G", [4, 8, 16, 32])
def test_lists_equal_the_oracle(ctx, B, G):
    sk, clips = _setup(B)
    n = 77
    lists = _lists(n, clips, seed=B * 100 + G)
    anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    anim.setLaunch(G)
    anim.setSamples(*lists)
    anim.update(1.0 / 30.0, ALL)
    exp = _expected(sk, clips, *lists)
    _check(anim, exp, f"B={B} G={G}")
    # no time is stepped: a second update gives the same bytes
    anim.update(0.5, ALL)
    _check(anim, exp, f"B={B} G={G}, second update")


def test_weight_and_time_edges_one_sample(ctx):
    """Every (weight, looped, time edge) combination as a one-sample list after a full-weight first sample of another clip."""
    sk, clips = _setup(64, seed=9)
    rows = []
    for w in WEIGHTS:
        for lo in (0, 1):
            for c in range(len(clips)):
                L = clips[c].length_ticks
                for t in (0, L - 1, L, L + 1, 3 * L + 7, 0xFFFFFFFF):
                    rows.append((c, t, w, lo))
    n = len(rows)
    offsets = np.arange(0, 2 * n + 1, 2, dtype=np.uint32)
    clip = np.empty(2 * n, np.uint32)
    tt = np.empty(2 * n, np.uint32)
    w = np.empty(2 * n, np.float32)
    lo = np.empty(2 * n, np.uint32)
    for i, (c, t, ww, l) in enumerate(rows):
        clip[2 * i], tt[2 * i], w[2 * i], lo[2 * i] = (c + 1) % len(clips), 1234, 1.0, 1
        clip[2 * i + 1], tt[2 * i + 1], w[2 * i + 1], lo[2 * i + 1] = c, t, ww, l
    anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    anim.setSamples(offsets, clip, tt, w, lo)
    anim.update(0.0, ALL)
    _check(anim, _expected(sk, clips, offsets, clip, tt, w, lo), "edges")


def test_layers_tie(ctx):
    """[base clip at weight 1, then the layers] as a list gives the bytes of clip mode + set_layers with the same entries (clamped times:
    the layer times stay below the clip length, where min(time, length) is the time itself)."""
    sk, clips = _setup(64, seed=5)
    n, K = 90, 3
    rng = np.random.default_rng(2)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    tt = (rng.random(n) * np.array([c.length_ticks for c in clips])[ci]).astype(np.uint32)
    lc = rng.integers(0, len(clips), (n, K)).astype(np.uint32)
    lt = (rng.random((n, K)) * np.array([c.length_ticks for c in clips])[lc]).astype(np.uint32)
    lw = np.array(WEIGHTS, np.float32)[rng.integers(0, len(WEIGHTS), (n, K))]
    layered = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    layered.setInstances(ci, tt)
    layered.setLayers(lc, lt, lw)
    layered.update(0.0, ALL)
    lists = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    offsets = np.arange(0, n * (K + 1) + 1, K + 1, dtype=np.uint32)
    clip = np.concatenate([ci[:, None], lc], 1).reshape(-1)
    time_ticks = np.concatenate([tt[:, None], lt], 1).reshape(-1)
    weight = np.concatenate([np.ones((n, 1), np.float32), lw], 1).reshape(-1)
    lists.setSamples(offsets, clip, time_ticks, weight, np.zeros(len(clip), np.uint32))
    lists.update(0.0, ALL)
    for get, what in ((lambda a: a.getPose()[0], "positions"), (lambda a: a.getPose()[1], "rotations"), (lambda a: a.getDualQuats(), "dual quaternions"),
                      (lambda a: a.getMatrices(), "matrices")):
        assert_bits_equal(get(lists), get(layered), f"list against layers: {what}")


def _system(ctx, sk, clips, n, seed, mode):
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    if mode == "clip":
        ci, tt = scenes.instance_times(n, clips, seed=seed)
        a.setInstances(ci, tt)
    else:
        a.setSamples(*_lists(n, clips, seed=seed))
    return a


@pytest.mark.parametrize("n_systems", [5, 70])
def test_update_many_mixed_modes(ctx, n_systems):
    """update_many over clip-mode and sample-list systems (over more than one launch at 70) equals per-system update, times included."""
    shapes = [_setup(64, seed=1), _setup(1, seed=2), _setup(196, seed=3)]
    many, one = [], []
    for s in range(n_systems):
        sk, clips = shapes[s % 3]
        mode = "list" if s % 2 == 0 else "clip"
        n = 3 + (s * 7) % 40
        many.append(_system(ctx, sk, clips, n, 40 + s, mode))
        one.append(_system(ctx, sk, clips, n, 40 + s, mode))
    lb.AnimationSystem.updateMany(many, 1.0 / 30.0, ALL)
    for a in one:
        a.update(1.0 / 30.0, ALL)
    for s, (a, b) in enumerate(zip(many, one)):
        p1, r1 = a.getPose()
        p2, r2 = b.getPose()
        assert_bits_equal(p1, p2, f"system {s}: positions")
        assert_bits_equal(r1, r2, f"system {s}: rotations")
        assert_bits_equal(a.getDualQuats(), b.getDualQuats(), f"system {s}: dual quaternions")
        assert_bits_equal(a.getMatrices(), b.getMatrices(), f"system {s}: matrices")
        if s % 2:
            assert_bits_equal(a.getTimes(), b.getTimes(), f"system {s}: times")
    sk, clips = shapes[0]
    assert_bits_equal(many[0].getPose()[0], _expected(sk, clips, *_lists(many[0].n, clips, seed=40))["pos"], "system 0 against the oracle")


def test_modes_switch(ctx):
    """set_samples -> sample-list mode (no time step, get_times / set_layers refused); set_instances -> clip mode as before."""
    sk, clips = _setup(64, seed=6)
    n = 40
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    ref = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    ci, tt = scenes.instance_times(n, clips, seed=8)
    ref.setInstances(ci, tt)
    ref.update(1.0 / 30.0, ALL)
    a.setInstances(ci, tt)
    lists = _lists(n, clips, seed=4)
    a.setSamples(*lists)
    for call in (lambda: a.getTimes(), lambda: a.setLayers(np.zeros((n, 1)), np.zeros((n, 1)), np.ones((n, 1)))):
        with pytest.raises(lb.LumixB200Error) as e:
            call()
        assert e.value.code == ERR_INVALID
    a.update(1.0 / 30.0, ALL)
    _check(a, _expected(sk, clips, *lists), "sample lists")
    a.setInstances(ci, tt)
    a.update(1.0 / 30.0, ALL)
    assert_bits_equal(a.getMatrices(), ref.getMatrices(), "clip mode after sample lists")
    assert_bits_equal(a.getTimes(), ref.getTimes(), "times after sample lists")


def test_refusals_change_nothing(ctx):
    sk, clips = _setup(64, seed=7)
    n = 20
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    lists = _lists(n, clips, seed=12)
    a.setSamples(*lists)
    a.update(0.0, ALL)
    exp = _expected(sk, clips, *lists)
    offsets, clip, tt, w, lo = lists
    bad_clip = clip.copy()
    bad_clip[-1] = len(clips)
    dec = offsets.copy()
    dec[5] = dec[6] + 1
    start = offsets + 1
    big = np.concatenate([offsets, offsets[-1:] + 1])
    for what, args in (("clip out of range", (offsets, bad_clip, tt, w, lo)), ("decreasing offsets", (dec, clip, tt, w, lo)),
                       ("offsets[0] != 0", (start, np.concatenate([clip, clip[:1]]), np.concatenate([tt, tt[:1]]), np.concatenate([w, w[:1]]),
                                            np.concatenate([lo, lo[:1]]))),
                       ("more instances than max_instances", (big, np.concatenate([clip, clip[:1]]), np.concatenate([tt, tt[:1]]),
                                                               np.concatenate([w, w[:1]]), np.concatenate([lo, lo[:1]])))):
        with pytest.raises(lb.LumixB200Error) as e:
            a.setSamples(*args)
        assert e.value.code == ERR_INVALID, what
        a.update(0.0, ALL)
        _check(a, exp, f"after a refused call ({what})")
    # an empty list set: every instance is the bind pose
    empty = np.zeros(n + 1, np.uint32)
    a.setSamples(empty, [], [], [], [])
    a.update(0.0, ALL)
    _check(a, _expected(sk, clips, empty, *(np.zeros(0, d) for d in (np.uint32, np.uint32, np.float32, np.uint32))), "empty lists")


def test_consumers(ctx):
    """skin, compute_relative, bone attachments and propagate_attached read a sample-list system's poses as a clip-mode system's."""
    sk, clips = _setup(64, seed=8)
    mesh = scenes.mesh(sk, 300)
    n = 24
    lists = _lists(n, clips, seed=13)
    a = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=n)
    a.setSamples(*lists)
    a.update(0.0, ALL)
    exp = _expected(sk, clips, *lists)
    a.skin()
    sk_out = a.getSkinned()
    for i in (0, 7, n - 1):
        assert_bits_equal(sk_out[i], po.skin_vertices(exp["mtx"][i], mesh.positions, mesh.weights, mesh.indices), f"skinned instance {i}")
    a.computeRelative()
    rp, rr = a.getRelativePose()
    for i in (0, 5, n - 1):
        p, r = po.pose_compute_relative(sk, exp["pos"][i], exp["rot"][i])
        assert_bits_equal(rp[i], p, f"relative positions {i}")
        assert_bits_equal(rr[i], r, f"relative rotations {i}")
    # bone attachments: the host call, the device call and the hierarchy's attachment rounds against the same bones of a clip-mode
    # system whose poses are the same bytes (a one-sample list at weight 1 is the clip mode's base clip)
    ci, tt = scenes.instance_times(n, clips[:2], seed=3)
    tt = np.minimum(tt, np.array([c.length_ticks for c in clips])[ci] - 1).astype(np.uint32)
    twin = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    twin.setInstances(ci, tt)
    twin.update(0.0, POSE)
    one = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    one.setSamples(np.arange(n + 1, dtype=np.uint32), ci, tt, np.ones(n, np.float32), np.zeros(n, np.uint32))
    one.update(0.0, POSE)
    assert_bits_equal(one.getPose()[0], twin.getPose()[0], "one-sample list against clip mode")
    m = 16
    rng = np.random.default_rng(1)
    inst = rng.integers(0, n, m).astype(np.uint32)
    bone = rng.integers(0, sk.bone_count, m).astype(np.uint32)
    rel = np.tile(np.array([0.1, 0.2, 0.3, 0, 0, 0, 1], np.float32), (m, 1))
    par = np.zeros(m, lb.TRANSFORM_DTYPE)
    par["rot"][:, 3] = 1
    par["scale"] = 1
    par["pos"] = rng.random((m, 3)) * 10
    scale = np.ones((m, 3), np.float32)
    assert_bits_equal(one.boneAttachments(inst, bone, rel, par, scale).view(np.uint32), twin.boneAttachments(inst, bone, rel, par, scale).view(np.uint32),
                      "bone attachments")
    out_one = _attached_frame(ctx, one, inst, bone)
    out_twin = _attached_frame(ctx, twin, inst, bone)
    assert_bits_equal(out_one.view(np.uint32), out_twin.view(np.uint32), "propagate_attached")


def _attached_frame(ctx, system, inst, bone):
    """A hierarchy of one parent entity with len(inst) attached children, propagated with the attachments on `system` -> globals."""
    m = len(inst)
    parents = np.array([-1] + [0] * m, np.int32)
    h = lb.Hierarchy(ctx, parents)
    loc = np.zeros(m + 1, lb.TRANSFORM_DTYPE)
    loc["rot"][:, 3] = 1
    loc["scale"] = 1
    h.setLocalTransforms(loc)
    root = np.zeros(m + 1, lb.TRANSFORM_DTYPE)  # globals of the roots (node 0), the other rows unread
    root["pos"] = (1.0, 2.0, 3.0)
    root["rot"][:, 3] = 1
    root["scale"] = 1
    h.setRootTransforms(root)
    h.setEntities(np.arange(m + 1, dtype=np.int32))
    rel = np.tile(np.array([0.1, 0.2, 0.3, 0, 0, 0, 1], np.float32), (m, 1))
    h.setAttachments(np.arange(1, m + 1, dtype=np.uint32), np.zeros(m, np.uint32), np.zeros(m, np.uint32), inst, bone, rel)
    h.propagateAttached([system], [1])
    g = h.getTransforms()
    h.close()
    return g
