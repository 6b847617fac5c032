"""lb200_animation_set_stacks (AnimationSystem.setStacks): the IK instructions of animators' blend stacks solved on the device, in stack
order with their samples.

Every case of ik_kat_inputs (tests/test_animation_ik_cpu.py) is held bit for bit to the restatement (oracle_pose_stack_ik, itself pinned
to the reference-run vectors of tests/golden/ik_kat.npz): absolute poses, dual quaternions and matrices, at every lane count, on 1-, 64-
and 196-bone skeletons, one with a 33-bone chain and one whose chains fold back by 180 degrees.  Instances without IK ops sit between
the IK instances inside each warp.  Then: update_many over IK, IK-free list and clip-mode systems against per-system updates, the pose
consumers (skin, bone attachments, propagate_attached) on an IK'd pose, set_samples dropping the ops, and the refusals."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from oracle import pyoracle as po
from bitexact import assert_bits_equal
from test_animation_ik_cpu import expected, ik_kat_inputs
from test_animation_stacks_gpu import _attached_frame

pytestmark = pytest.mark.gpu

DQ, MTX, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_MATRIX, lb.PALETTE_POSE
ALL = DQ | MTX | POSE
ERR_INVALID = lb._lib.ERR_INVALID
INPUTS = ik_kat_inputs()


@pytest.fixture(scope="module")
def ctx():
    c = lb.Context(0)
    yield c
    c.close()


def _stacks(cases, plain_every=3):
    """The cases as instances, with an instance that has the case's samples but no IK op after every `plain_every` of them (IK and IK-free
    instances share warps; None: the cases alone) -> (setStacks arguments, [case per instance])."""
    inst = []
    for k, case in enumerate(cases):
        inst.append(case)
        if plain_every and k % plain_every == 0:
            slot, weight, t, looped = case[:4]
            inst.append((slot, weight, t, looped, *(np.zeros(0, d) for d in (np.uint32, np.uint32, np.uint32, np.float32)), np.zeros((0, 3), np.float32)))
    cat = lambda j, d: np.concatenate([c[j] for c in inst]).astype(d) if inst else np.zeros(0, d)  # noqa: E731
    offsets = np.concatenate([[0], np.cumsum([len(c[0]) for c in inst])]).astype(np.uint32)
    ik_offsets = np.concatenate([[0], np.cumsum([len(c[4]) for c in inst])]).astype(np.uint32)
    args = (offsets, cat(0, np.uint32), cat(2, np.uint32), cat(1, np.float32), cat(3, np.uint32), ik_offsets, cat(4, np.uint32), cat(5, np.uint32),
            cat(6, np.uint32), cat(7, np.float32), np.concatenate([c[8].reshape(-1, 3) for c in inst]).astype(np.float32))
    return args, inst


def _expected(sk, clips, inst):
    n, B = len(inst), sk.bone_count
    out = dict(pos=np.empty((n, B, 3), np.float32), rot=np.empty((n, B, 4), np.float32), dq=np.empty((n, B, 8), np.float32), mtx=np.empty((n, B, 16), np.float32))
    for i, case in enumerate(inst):
        out["pos"][i], out["rot"][i] = expected(sk, clips, case)
        out["dq"][i], out["mtx"][i] = po.palettes(sk, out["pos"][i], out["rot"][i])
    return out


def _check(anim, exp, what):
    p, r = anim.getPose()
    assert_bits_equal(p, exp["pos"], f"{what}: pose positions")
    assert_bits_equal(r, exp["rot"], f"{what}: pose rotations")
    assert_bits_equal(anim.getDualQuats(), exp["dq"], f"{what}: dual quaternions")
    assert_bits_equal(anim.getMatrices(), exp["mtx"], f"{what}: matrices")


@pytest.mark.parametrize("name", list(INPUTS))
@pytest.mark.parametrize("G", [4, 8, 16, 32])
def test_stacks_equal_the_oracle(ctx, name, G):
    sk, clips, cases = INPUTS[name]
    args, inst = _stacks(cases)
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=len(inst))
    a.setLaunch(G, 0)
    a.setStacks(*args)
    a.update(0.0, ALL)
    _check(a, _expected(sk, clips, inst), f"{name} G={G}")
    a.close()


def test_vectors_through_the_device(ctx):
    """The device against the reference-run vectors directly, not only through the restatement."""
    import os
    kat = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ik_kat.npz"))
    for name, (sk, clips, cases) in INPUTS.items():
        args, inst = _stacks(cases, plain_every=None)
        a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=len(inst))
        a.setStacks(*args)
        a.update(0.0, POSE)
        p, r = a.getPose()
        for k in range(len(cases)):
            assert_bits_equal(p[k], kat[f"{name}_c{k}_pos"], f"{name} case {k}: positions")
            assert_bits_equal(r[k], kat[f"{name}_c{k}_rot"], f"{name} case {k}: rotations")
        a.close()


def _three_systems(ctx, seed_name="b64"):
    """An IK system, an IK-free list system and a clip-mode system of the same skeleton."""
    sk, clips, cases = INPUTS[seed_name]
    args, inst = _stacks(cases)
    n = len(inst)
    ik = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    ik.setStacks(*args)
    plain = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    plain.setSamples(*args[:5])
    clip = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    rng = np.random.default_rng(2)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    clip.setInstances(ci, (rng.random(n) * np.array([c.length_ticks for c in clips])[ci]).astype(np.uint32))
    return [ik, plain, clip]


def _outputs(systems):
    return [(s.getPose()[0].copy(), s.getPose()[1].copy(), s.getDualQuats().copy(), s.getMatrices().copy()) for s in systems]


def test_update_many_mixed(ctx):
    solo = _three_systems(ctx)
    for s in solo:
        s.update(1.0 / 30.0, ALL)
    many = _three_systems(ctx)
    lb.AnimationSystem.updateMany(many, 1.0 / 30.0, ALL)
    for k, (a, b) in enumerate(zip(_outputs(solo), _outputs(many))):
        for x, y, what in zip(a, b, ("positions", "rotations", "dual quaternions", "matrices")):
            assert_bits_equal(y, x, f"system {k}: {what}")
    assert_bits_equal(many[2].getTimes(), solo[2].getTimes(), "clip-mode times")
    # the IK-free pair in one launch runs the kernel without IK and gives the same bytes
    pair = _three_systems(ctx)[1:]
    lb.AnimationSystem.updateMany(pair, 1.0 / 30.0, ALL)
    for k, (a, b) in enumerate(zip(_outputs(solo[1:]), _outputs(pair))):
        for x, y in zip(a, b):
            assert_bits_equal(y, x, f"IK-free system {k}")
    for s in solo + many + pair:
        s.close()


def test_consumers(ctx):
    """skin, bone attachments and propagate_attached read an IK'd pose."""
    from lumixengine_b200 import scenes
    sk, clips, cases = INPUTS["b64"]
    args, inst = _stacks(cases)
    n = len(inst)
    mesh = scenes.mesh(sk, 300)
    a = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=n)
    a.setStacks(*args)
    a.update(0.0, ALL)
    exp = _expected(sk, clips, inst)
    a.skin()
    out = a.getSkinned()
    for i in (0, 5, n - 1):
        assert_bits_equal(out[i], po.skin_vertices(exp["mtx"][i], mesh.positions, mesh.weights, mesh.indices), f"skinned instance {i}")
    ik_inst = np.array([i for i, c in enumerate(inst) if len(c[4]) and c[7].max() >= 0.001], np.uint32)[:16]
    bone = np.array([int(inst[i][5][0]) for i in ik_inst], np.uint32)  # the leaf of the instance's first op
    m = len(ik_inst)
    rel = np.tile(np.array([0.1, 0.2, 0.3, 0, 0, 0, 1], np.float32), (m, 1))
    par = np.zeros(m, lb.TRANSFORM_DTYPE)
    par["pos"] = (1.0, 2.0, 3.0)
    par["rot"][:, 3] = 1
    par["scale"] = 1
    scale = np.ones((m, 3), np.float32)
    got = a.boneAttachments(ik_inst, bone, rel, par, scale)
    bone7 = np.concatenate([exp["pos"][ik_inst, bone], exp["rot"][ik_inst, bone]], 1).astype(np.float32)
    want = po.bone_attachments(np.ascontiguousarray(par).view(np.uint8).reshape(m, 56), bone7, rel, scale).view(lb.TRANSFORM_DTYPE).reshape(-1)
    assert_bits_equal(got["pos"], want["pos"], "bone attachments: positions")
    assert_bits_equal(got["rot"], want["rot"], "bone attachments: rotations")
    g = _attached_frame(ctx, a, ik_inst, bone)
    assert_bits_equal(g["pos"][1:], got["pos"], "propagate_attached: positions")
    assert_bits_equal(g["rot"][1:], got["rot"], "propagate_attached: rotations")
    a.close()


def test_set_samples_drops_the_ik_ops(ctx):
    sk, clips, cases = INPUTS["c33"]
    args, inst = _stacks(cases)
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=len(inst))
    a.setStacks(*args)
    a.setSamples(*args[:5])
    a.update(0.0, ALL)
    plain = [(*c[:4], *(np.zeros(0, d) for d in (np.uint32, np.uint32, np.uint32, np.float32)), np.zeros((0, 3), np.float32)) for c in inst]
    _check(a, _expected(sk, clips, plain), "set_samples after set_stacks")
    a.close()


def test_refusals_change_nothing(ctx):
    sk, clips, cases = INPUTS["c33"]
    args, inst = _stacks(cases)
    n = len(inst)
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    a.setStacks(*args)
    a.update(0.0, ALL)
    exp = _expected(sk, clips, inst)
    _check(a, exp, "before the refusals")
    off, clip, t, w, lo, iko, after, leaf, bones, alpha, tgt = args
    k = int(np.nonzero(np.diff(iko) > 0)[0][0])  # an instance with IK ops
    j = int(iko[k])

    def bad(**kw):
        a2 = dict(off=off, clip=clip, t=t, w=w, lo=lo, iko=iko, after=after, leaf=leaf, bones=bones, alpha=alpha, tgt=tgt)
        for key, v in kw.items():
            a2[key] = v
        return tuple(a2[x] for x in ("off", "clip", "t", "w", "lo", "iko", "after", "leaf", "bones", "alpha", "tgt"))

    def edit(arr, i, v):
        c = arr.copy()
        c[i] = v
        return c

    refusals = {
        "ik_offsets[0] != 0": bad(iko=edit(iko, 0, 1)),
        "decreasing ik_offsets": bad(iko=edit(iko, len(iko) - 2, iko[-1] + 1)),
        "after past the list": bad(after=edit(after, j, off[k + 1] - off[k] + 1)),
        "leaf out of range": bad(leaf=edit(leaf, j, sk.bone_count)),
        "bone count 0": bad(bones=edit(bones, j, 0)),
        "bone count 33": bad(bones=edit(bones, j, 33)),
        "chain leaves the skeleton": bad(leaf=edit(leaf, j, 0), bones=edit(bones, j, 2)),  # bone 0 is the root
        "clip out of range": bad(clip=edit(clip, 0, len(clips))) if len(clip) else None,
    }
    # decreasing `after` inside an instance: an instance with two ops at different positions
    two = [i for i in range(n) if iko[i + 1] - iko[i] == 2 and after[iko[i]] != after[iko[i] + 1]]
    if two:
        i = two[0]
        refusals["after decreasing"] = bad(after=edit(edit(after, int(iko[i]), after[iko[i] + 1]), int(iko[i]) + 1, after[iko[i]]))
    assert len(refusals) >= 8
    for what, r in refusals.items():
        if r is None:
            continue
        with pytest.raises(lb.LumixB200Error) as e:
            a.setStacks(*r)
        assert e.value.code == ERR_INVALID, what
        a.update(0.0, ALL)
        _check(a, exp, f"after the refusal '{what}'")
    a.close()
