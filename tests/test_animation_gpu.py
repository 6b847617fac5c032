"""GPU parity of pose evaluation, skinning palettes and CPU-path skinning against the oracle.

The kernels keep the reference's op order without FMA, so every pose, palette and skinned vertex must equal the oracle's bit
for bit (DESIGN §2).  north_star's 1e-5 relative tolerance for skin matrices is the product's promise, not what these tests allow.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from bitexact import assert_bits_equal as _close

pytestmark = pytest.mark.gpu


def _setup(ctx, n_bones, n_clips, n_inst, n_verts=0, seed=0, **clip_kw):
    sk = scenes.skeleton(n_bones, seed=seed + 4)
    clips = [scenes.clip(sk, frames=30 + 7 * i, fps=30.0 if i % 2 == 0 else 24.0, seed=seed + 10 + i, **clip_kw) for i in range(n_clips)]
    mesh = scenes.mesh(sk, n_verts, seed=seed + 6) if n_verts else None
    anim = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=n_inst)
    ci, tt = scenes.instance_times(n_inst, clips, seed=seed + 7)
    anim.setInstances(ci, tt)
    return sk, clips, mesh, anim, ci, tt


@pytest.mark.parametrize("n_bones,n_clips,n_inst", [(64, 4, 3000), (5, 1, 33), (196, 2, 500), (1, 1, 10)])
def test_pose_and_palettes_match_oracle(ctx, oracle, n_bones, n_clips, n_inst):
    sk, clips, _, anim, ci, tt = _setup(ctx, n_bones, n_clips, n_inst, seed=n_bones)
    anim.update(0.0, lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE)
    exp = oracle.animate_instances(sk, clips, ci, tt)
    pos, rot = anim.getPose()
    _close(pos, exp["pos"], "pose.pos"); _close(rot, exp["rot"], "pose.rot")
    _close(anim.getDualQuats(), exp["dq"], "dual quats"); _close(anim.getMatrices(), exp["mtx"], "matrices")
    assert np.array_equal(anim.getTimes(), tt)  # time_delta == 0 leaves the animables' time alone


def test_clip_edges_and_bit_widths(ctx, oracle):
    """t = 0, t = length-1, times beyond the clip (clamped by frame_count - 1e-5), odd bit widths (11..16 + 57-bit tracks)."""
    sk = scenes.skeleton(24, seed=2)
    clips = [scenes.clip(sk, frames=17, fps=30.0, seed=3, pos_bits=(11, 13, 16), rot_bits=(12, 14, 16), const_fraction=0.0),
             scenes.clip(sk, frames=60, fps=60.0, seed=4, pos_bits=(16, 16, 16), rot_bits=(16, 16, 16), const_fraction=0.5),
             scenes.clip(sk, frames=2, fps=1.0, seed=5, pos_bits=(5, 3, 7), rot_bits=(9, 9, 9), const_fraction=1.0)]
    anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=64)
    ci, tt = [], []
    for c, clip in enumerate(clips):
        L = clip.length_ticks
        for t in (0, 1, L // 2, L - 1, L, L + 5000, 2 ** 31):
            ci.append(c); tt.append(t)
    ci, tt = np.array(ci, np.uint32), np.array(tt, np.uint32)
    anim.setInstances(ci, tt)
    anim.update(0.0, lb.PALETTE_DUAL_QUAT | lb.PALETTE_POSE)
    exp = oracle.animate_instances(sk, clips, ci, tt, want=("pos", "rot", "dq"))
    pos, rot = anim.getPose()
    _close(pos, exp["pos"], "pos"); _close(rot, exp["rot"], "rot"); _close(anim.getDualQuats(), exp["dq"], "dq")


def test_time_advance(ctx, oracle):
    sk, clips, _, anim, ci, tt = _setup(ctx, 16, 3, 2000, seed=40)
    for dt in (1.0 / 60.0, 0.5, 3.7, -0.25):
        anim.setInstances(ci, tt)
        anim.update(dt, lb.PALETTE_DUAL_QUAT)
        got = anim.getTimes()
        # animation_module.cpp:458-469, both signs of time_delta (the oracle is pinned against the reference's own Time operators)
        exp = np.array([oracle.time_advance(t, dt, clips[c].fps, clips[c].frame_count) for c, t in zip(ci, tt)], np.uint32)
        assert np.array_equal(got, exp)


def test_skinning_matches_oracle(ctx, oracle):
    sk, clips, mesh, anim, ci, tt = _setup(ctx, 64, 2, 37, n_verts=1777, seed=70)
    anim.update(0.0, lb.PALETTE_MATRIX)
    anim.skin()
    got = anim.getSkinned()
    mtx = anim.getMatrices()
    for i in range(len(ci)):  # 37 instances: the last skin group (32..36) is partial
        exp = oracle.skin_vertices(mtx[i], mesh.positions, mesh.weights, mesh.indices)
        _close(got[i], exp, f"skinned verts of instance {i}")
    # checksum of the device buffer equals the checksum of what was read back
    assert anim.skinnedChecksum() == int(got.view(np.uint32).astype(np.uint64).sum())


def test_c4_size_properties(ctx):
    """Config 4 shapes at reduced instance count that still exceeds L2 (20 k x 64 bones x 5 k verts = 1.2 GB out):
    rigid property — with every weight on one bone, skinning equals the bone matrix applied to the vertex."""
    sk = scenes.skeleton(64)
    clips = [scenes.clip(sk, frames=60, seed=s) for s in (1, 2, 3, 4)]
    mesh = scenes.mesh(sk, 5000)
    mesh.weights[:] = 0
    mesh.weights[:, 0] = 1.0
    n = 20_000
    anim = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=n)
    ci, tt = scenes.instance_times(n, clips)
    anim.setInstances(ci, tt)
    anim.update(1.0 / 30.0, lb.PALETTE_MATRIX | lb.PALETTE_DUAL_QUAT)
    anim.skin()
    for first in (0, n - 3):
        m = anim.getMatrices(first, 3).reshape(3, 64, 4, 4)  # [col][row]
        v = anim.getSkinned(first, 3)
        mv = m[:, mesh.indices[:, 0]]  # (3, V, 4, 4)
        p = mesh.positions
        exp = mv[:, :, 0, :3] * p[None, :, 0:1] + mv[:, :, 1, :3] * p[None, :, 1:2] + mv[:, :, 2, :3] * p[None, :, 2:3] + mv[:, :, 3, :3]
        assert np.allclose(v, exp, rtol=1e-5, atol=1e-5)
    # dual quaternion palette: real part is a unit quaternion, dual part orthogonal to it
    dq = anim.getDualQuats(0, 100)
    assert np.allclose(np.linalg.norm(dq[..., :4], axis=-1), 1.0, atol=1e-4)
    assert np.all(np.abs((dq[..., :4] * dq[..., 4:]).sum(axis=-1)) < 1e-3)


def test_compute_relative_and_blend_match_oracle(ctx, oracle):
    """Pose::computeRelative (pose.cpp:136-146) and Pose::blend (pose.cpp:30-41) batched over instances, against the oracle."""
    n_inst = 700
    sk, clips, _, a, ci, tt = _setup(ctx, 48, 3, n_inst, seed=21)
    b = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n_inst)
    ci_b, tt_b = scenes.instance_times(n_inst, clips, seed=99)
    b.setInstances(ci_b, tt_b)
    for s in (a, b):
        s.update(0.0, lb.PALETTE_POSE)
        s.computeRelative()
    abs_a, abs_b = a.getPose(), b.getPose()
    rel_a, rel_b = a.getRelativePose(), b.getRelativePose()
    for i in (0, 1, 17, n_inst - 1):
        ep, er = oracle.pose_compute_relative(sk, abs_a[0][i], abs_a[1][i])
        _close(rel_a[0][i], ep, "relative pos"); _close(rel_a[1][i], er, "relative rot")
    # blend in both spaces, several weights (0.0005 must leave the pose untouched; 1.7 clamps to 1)
    for w, relative in ((0.0005, False), (0.3, False), (0.5, True), (1.7, True)):
        a.blendPose(b, w, relative=relative)
        cur = a.getRelativePose() if relative else a.getPose()
        src_a, src_b = (rel_a, rel_b) if relative else (abs_a, abs_b)
        for i in (0, 5, n_inst - 1):
            ep, er = oracle.pose_blend(src_a[0][i], src_a[1][i], src_b[0][i], src_b[1][i], w)
            _close(cur[0][i], ep, f"blend pos w={w}"); _close(cur[1][i], er, f"blend rot w={w}")
        if relative:
            rel_a = cur
        else:
            abs_a = cur
    a.close(); b.close()


def test_blend_layers_match_oracle(ctx, oracle):
    """Weighted sample stack per instance (Animation::getRelativePose with ctx.weight, animation.cpp:117-204, 294-311): base clip, then
    layers with weights below and above the 0.9999 switch, clips with constant tracks (which blend) and untracked bones (which do not)."""
    n_inst, n_layers = 300, 3
    sk, clips, _, anim, ci, tt = _setup(ctx, 40, 4, n_inst, seed=33, const_fraction=0.3)
    rng = np.random.default_rng(8)
    lci = rng.integers(0, len(clips), (n_inst, n_layers)).astype(np.uint32)
    ltt = np.stack([rng.integers(0, clips[c].length_ticks, n_inst) for c in range(n_layers)], axis=1).astype(np.uint32)
    lw = rng.random((n_inst, n_layers)).astype(np.float32)
    lw[::7, 1] = 1.0       # replacement instead of blending
    lw[::11, 0] = 0.99995  # just above the switch
    lw[::13, 2] = 0.0
    # one layer first, then all of them: the second call replaces the layer tables with larger ones
    for k_used in (1, n_layers):
        anim.setLayers(lci[:, :k_used], ltt[:, :k_used], lw[:, :k_used])
        anim.update(0.0, lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE)
        pos, rot = anim.getPose()
        dq, mtx = anim.getDualQuats(), anim.getMatrices()
        for i in list(range(0, n_inst, 7)) + [1, 2, n_inst - 1]:
            p, r = oracle.pose_evaluate(sk, clips[ci[i]], tt[i], compute_absolute=False)
            for k in range(k_used):
                p, r = oracle.pose_evaluate(sk, clips[lci[i, k]], ltt[i, k], weight=float(lw[i, k]), start_from_bind=False, compute_absolute=False, pos=p, rot=r)
            p, r = oracle.pose_compute_absolute(sk, p, r)
            edq, emtx = oracle.palettes(sk, p, r)
            _close(pos[i], p, "layered pose.pos"); _close(rot[i], r, "layered pose.rot"); _close(dq[i], edq, "layered dq"); _close(mtx[i], emtx, "layered mtx")
    # removing the layers gives the plain single-clip result again
    anim.setLayers(None, None, None)
    anim.update(0.0, lb.PALETTE_POSE)
    exp = oracle.animate_instances(sk, clips, ci, tt)
    _close(anim.getPose()[0], exp["pos"], "pose.pos after removing layers")
    anim.close()


def test_random_skeletons_and_clips(ctx, oracle):
    """Randomised parity run: 1..196 bones, 1..90 frames, 5..18-bit channels, any share of constant tracks, several clips per system,
    times inside / at / beyond the clip end; pose, both palettes and the advanced time against the oracle."""
    rng = np.random.default_rng(123)
    for trial in range(10):
        bones = int(rng.choice([1, 2, 3, 5, 16, 33, 64, 100, 196]))
        sk = scenes.skeleton(bones, seed=800 + trial)
        clips = []
        for c in range(int(rng.integers(1, 4))):
            pb = tuple(int(x) for x in rng.integers(5, 19, 3))
            rb = tuple(int(x) for x in rng.integers(5, 19, 3))
            clips.append(scenes.clip(sk, frames=int(rng.integers(1, 91)), fps=float(rng.choice([1.0, 24.0, 30.0, 59.94])), seed=900 + 10 * trial + c,
                                     pos_bits=pb, rot_bits=rb, const_fraction=float(rng.choice([0.0, 0.25, 1.0]))))
        n_inst = int(rng.integers(1, 400))
        ci = rng.integers(0, len(clips), n_inst).astype(np.uint32)
        lengths = np.array([c.length_ticks for c in clips], np.int64)
        tt = (rng.random(n_inst) * (lengths[ci] + 3)).astype(np.uint32)  # a few at or past the end: clamped by frame_count - 1e-5
        tt[:3] = [0, 1, int(lengths[ci[2 % n_inst]])][:min(3, n_inst)] if n_inst >= 3 else tt[:3]
        anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n_inst)
        anim.setInstances(ci, tt)
        dt = float(rng.choice([0.0, 1.0 / 60.0, 0.75]))
        anim.update(dt, lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE)
        exp = oracle.animate_instances(sk, clips, ci, tt)
        pos, rot = anim.getPose()
        _close(pos, exp["pos"], f"trial {trial} pose.pos"); _close(rot, exp["rot"], f"trial {trial} pose.rot")
        _close(anim.getDualQuats(), exp["dq"], f"trial {trial} dual quats"); _close(anim.getMatrices(), exp["mtx"], f"trial {trial} matrices")
        want = np.array([oracle.time_advance(t, dt, clips[c].fps, clips[c].frame_count) for c, t in zip(ci, tt)], np.uint32)
        assert np.array_equal(anim.getTimes(), want), trial
        anim.close()


def test_bone_attachments_match_oracle(ctx, oracle):
    """updateBoneAttachment batched (render_module.cpp:377-405, SURVEY 8f N4): entities following bones of posed instances."""
    n_inst = 200
    sk, clips, _, anim, ci, tt = _setup(ctx, 40, 2, n_inst, seed=61)
    anim.update(0.0, lb.PALETTE_POSE)
    pos, rot = anim.getPose()
    rng = np.random.default_rng(4)
    n = 1500
    inst = rng.integers(0, n_inst, n).astype(np.uint32)
    bone = rng.integers(0, 40, n).astype(np.uint32)
    rel = np.concatenate([(rng.normal(size=(n, 3)) * 0.5).astype(np.float32), scenes.random_unit_quats(rng, n)], axis=1).astype(np.float32)
    par = np.zeros(n, lb.TRANSFORM_DTYPE)
    par["pos"] = rng.normal(size=(n, 3)) * 5000.0
    par["rot"] = scenes.random_unit_quats(rng, n)
    par["scale"] = (0.5 + rng.random((n, 3))).astype(np.float32)
    scale = (0.5 + rng.random((n, 3))).astype(np.float32)
    got = anim.boneAttachments(inst, bone, rel, par, scale)
    bone7 = np.concatenate([pos[inst, bone], rot[inst, bone]], axis=1).astype(np.float32)
    exp = oracle.bone_attachments(np.ascontiguousarray(par).view(np.uint8).reshape(n, 56), bone7, rel, scale).view(lb.TRANSFORM_DTYPE).reshape(-1)
    assert np.array_equal(got["pos"], exp["pos"]) and np.array_equal(got["rot"].view(np.uint32), exp["rot"].view(np.uint32))
    assert np.array_equal(got["scale"], exp["scale"])
    anim.close()


def test_c4_100k_x64_palettes_equal_oracle_at_full_size(ctx, oracle):
    """BASELINE configs[3] at its stated size: 100 k instances x 64 bones — absolute poses, dual-quaternion and matrix palettes of every
    instance against the C restatement of updateAnimable + computeSkeletonDualQuats + computeSkinMatrices, bit for bit."""
    sk = scenes.skeleton(64)
    clips = [scenes.clip(sk, frames=60, seed=s) for s in (1, 2, 3, 4)]
    n = 100_000
    anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    ci, tt = scenes.instance_times(n, clips)
    anim.setInstances(ci, tt)
    anim.update(0.0, lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE)
    exp = oracle.animate_instances(sk, clips, ci, tt)
    pos, rot = anim.getPose()
    _close(pos, exp["pos"], "pose.pos"); _close(rot, exp["rot"], "pose.rot")
    _close(anim.getDualQuats(), exp["dq"], "dual quats"); _close(anim.getMatrices(), exp["mtx"], "matrices")
    anim.close()
