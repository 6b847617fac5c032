"""The pose, relative / blend and skinning kernels at every launch shape they have, bit for bit against the oracle.

pose_palette_kernel<G> runs G lanes per instance (128 / G instances per block); the default is 8, and setLaunch reaches 4, 16 and
32.  skin_kernel<group> stages `group` instance palettes per block; the default is 8, and setLaunch reaches 4 and 16.  The skeletons
cover the shapes that move the kernels' edges: padding of Bp (1-3 bones), no non-root level, several roots, a level wider than 32
lanes, the deepest chain, the 4-lane shared-memory fallback (192 / 196 bones) and an irregular tree.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from bitexact import assert_bits_equal

pytestmark = pytest.mark.gpu

ALL_PALETTES = lb.PALETTE_DUAL_QUAT | lb.PALETTE_MATRIX | lb.PALETTE_POSE


def _random_tree(n, seed):
    rng = np.random.default_rng(seed)
    return [-1] + [int(rng.integers(0, i)) for i in range(1, n)]


def _five_root_forest():
    # 5 roots, 8 children each (a level of 40 bones), then 25 bones under random earlier non-roots
    rng = np.random.default_rng(11)
    parents = [-1] * 5 + [r for r in range(5) for _ in range(8)]
    for i in range(len(parents), 70):
        parents.append(int(rng.integers(5, i)))
    return parents


SHAPES = {
    "1": [-1],
    "2": [-1, 0],
    "3": [-1, 0, 1],
    "all_roots": [-1] * 7,
    "five_roots": _five_root_forest(),
    "star196": [-1] + [0] * 195,
    "chain196": [-1] + list(range(195)),
    "chain192": [-1] + list(range(191)),
    "random150": _random_tree(150, 5),
    "c4_64": None,  # scenes.skeleton's own shape
}


def _skeleton(name):
    parents = SHAPES[name]
    return scenes.skeleton(64, seed=4) if parents is None else scenes.skeleton(seed=len(parents), parents=parents)


def _clips(sk):
    return [scenes.clip(sk, frames=13, fps=30.0, seed=21, const_fraction=0.3),
            scenes.clip(sk, frames=40, fps=24.0, seed=22, pos_bits=(11, 14, 16), rot_bits=(12, 15, 16), const_fraction=0.3)]


def _times(n, clips, seed):
    """Clip index and time of n instances: 0, inside, one tick before the end, at the end and past it, then random inside."""
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    lengths = np.array([c.length_ticks for c in clips], np.int64)[ci]
    tt = (rng.random(n) * lengths).astype(np.int64)
    edges = [lambda L: 0, lambda L: L - 1, lambda L: L, lambda L: L + 4000, lambda L: L // 3]
    for k, f in enumerate(edges[:n]):
        tt[k] = f(lengths[k])
    return ci, tt.astype(np.uint32)


def _expected_lanes(lanes, bones):
    if lanes == 0:
        return 8
    if lanes == 4 and bones > 192:
        return 8  # 32 poses of 196 bones do not fit in shared memory
    return lanes


def _check_update(oracle, anim, sk, clips, ci, tt, dt, what):
    exp = oracle.animate_instances(sk, clips, ci, tt)
    pos, rot = anim.getPose()
    assert_bits_equal(pos, exp["pos"], f"{what}: pose.pos")
    assert_bits_equal(rot, exp["rot"], f"{what}: pose.rot")
    assert_bits_equal(anim.getDualQuats(), exp["dq"], f"{what}: dual quats")
    assert_bits_equal(anim.getMatrices(), exp["mtx"], f"{what}: matrices")
    want = np.array([oracle.time_advance(t, dt, clips[c].fps, clips[c].frame_count) for c, t in zip(ci, tt)], np.uint32)
    assert np.array_equal(anim.getTimes(), want), f"{what}: advanced times"


def _check_layers(oracle, anim, sk, clips, ci, tt, what):
    """Two blend layers per instance, weights below, at and above the 0.9999 switch, against the layered pose_evaluate chain."""
    n = len(ci)
    rng = np.random.default_rng(n)
    lci = rng.integers(0, len(clips), (n, 2)).astype(np.uint32)
    ltt = np.stack([(rng.random(n) * np.array([clips[c].length_ticks for c in lci[:, k]])).astype(np.uint32) for k in range(2)], axis=1)
    lw = np.empty((n, 2), np.float32)
    lw[:, 0] = rng.random(n).astype(np.float32) * np.float32(0.9)
    lw[:, 1] = np.array([0.5, 1.0, 0.99995, 0.9999, 0.25], np.float32)[np.arange(n) % 5]
    anim.setInstances(ci, tt)
    anim.setLayers(lci, ltt, lw)
    anim.update(0.0, ALL_PALETTES)
    pos, rot = anim.getPose()
    dq, mtx = anim.getDualQuats(), anim.getMatrices()
    for i in range(n):
        p, r = oracle.pose_evaluate(sk, clips[ci[i]], tt[i], compute_absolute=False)
        for k in range(2):
            p, r = oracle.pose_evaluate(sk, clips[lci[i, k]], ltt[i, k], weight=float(lw[i, k]), start_from_bind=False, compute_absolute=False, pos=p, rot=r)
        p, r = oracle.pose_compute_absolute(sk, p, r)
        edq, emtx = oracle.palettes(sk, p, r)
        assert_bits_equal(pos[i], p, f"{what}: layered pose.pos of instance {i}")
        assert_bits_equal(rot[i], r, f"{what}: layered pose.rot of instance {i}")
        assert_bits_equal(dq[i], edq, f"{what}: layered dq of instance {i}")
        assert_bits_equal(mtx[i], emtx, f"{what}: layered mtx of instance {i}")
    anim.setLayers(None, None, None)


@pytest.mark.parametrize("lanes", [0, 4, 8, 16, 32])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_pose_and_palettes_every_lane_count(ctx, oracle, shape, lanes):
    sk = _skeleton(shape)
    clips = _clips(sk)
    G = _expected_lanes(lanes, sk.bone_count)
    per_block = 128 // G
    counts = [1, per_block - 1, per_block, per_block + 1, 333]
    anim = lb.AnimationSystem(ctx, sk, clips, None, max_instances=max(counts))
    anim.setLaunch(pose_lanes=lanes)
    for k, n in enumerate(counts):
        ci, tt = _times(n, clips, seed=100 * k + sk.bone_count)
        dt = (1.0 / 60.0, 0.75, -0.3, 2.5, 1.0 / 30.0)[k]
        anim.setInstances(ci, tt)
        anim.update(dt, ALL_PALETTES)
        assert anim.lastLaunch()[0] == G
        _check_update(oracle, anim, sk, clips, ci, tt, dt, f"{shape}, lanes {lanes}, {n} instances")
        if n == per_block + 1:
            _check_layers(oracle, anim, sk, clips, ci, tt, f"{shape}, lanes {lanes}, {n} instances")
    anim.close()


@pytest.mark.parametrize("shape", ["five_roots", "star196", "chain196"])
def test_relative_and_blend_every_instance(ctx, oracle, shape):
    sk = _skeleton(shape)
    clips = _clips(sk)
    n = 67
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    b = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    for s, seed in ((a, 1), (b, 2)):
        s.setInstances(*_times(n, clips, seed))
        s.update(0.0, lb.PALETTE_POSE)
        s.computeRelative()
    abs_a, abs_b = a.getPose(), b.getPose()
    rel_a, rel_b = a.getRelativePose(), b.getRelativePose()
    for i in range(n):
        ep, er = oracle.pose_compute_relative(sk, abs_a[0][i], abs_a[1][i])
        assert_bits_equal(rel_a[0][i], ep, f"{shape}: relative pos of instance {i}")
        assert_bits_equal(rel_a[1][i], er, f"{shape}: relative rot of instance {i}")
    B = sk.bone_count
    for relative in (False, True):
        cur_a, src_b = (rel_a, rel_b) if relative else (abs_a, abs_b)
        for w in (0.0005, 0.3, 1.7):
            a.blendPose(b, w, relative=relative)
            got = a.getRelativePose() if relative else a.getPose()
            # Pose::blend is bone by bone: the oracle takes every instance's bones as one pose
            ep, er = oracle.pose_blend(cur_a[0].reshape(-1, 3), cur_a[1].reshape(-1, 4), src_b[0].reshape(-1, 3), src_b[1].reshape(-1, 4), w)
            space = "relative" if relative else "absolute"
            assert_bits_equal(got[0], ep.reshape(n, B, 3), f"{shape}: {space} blend pos w={w}")
            assert_bits_equal(got[1], er.reshape(n, B, 4), f"{shape}: {space} blend rot w={w}")
            cur_a = got
    a.close(); b.close()


def _edge_mesh(sk, n_vertices, seed):
    """scenes.mesh with edge vertices spread over it: all-zero weights, -0.0 weights, weight 1 on the last bone, one bone index in
    all four slots."""
    m = scenes.mesh(sk, n_vertices, seed=seed)
    last = sk.bone_count - 1
    rows = [(np.zeros(4), None), (np.full(4, -0.0), None), (np.array([1.0, 0, 0, 0]), [last, 0, 0, 0]),
            (np.array([0.1, 0.2, 0.3, 0.4]), [last // 2] * 4), (np.array([0, 0, 0, 1.0]), [0, 0, 0, last])]
    for k, (w, idx) in enumerate(rows):
        v = (k * 61) % n_vertices
        m.weights[v] = w.astype(np.float32)
        if idx is not None:
            m.indices[v] = idx
    return m


@pytest.mark.parametrize("group", [0, 4, 16])
@pytest.mark.parametrize("bones", [1, 64, 196])
def test_skinning_every_group_and_instance(ctx, oracle, bones, group):
    sk = scenes.skeleton(bones, seed=bones) if bones == 64 else scenes.skeleton(seed=bones, parents=[-1] + list(range(bones - 1)))
    clips = _clips(sk)
    g = group or 8
    counts = [2 * g, 2 * g + 1, 3 * g - 1, 3]  # n mod group = 0, 1, group - 1, and fewer instances than one group
    for n_vertices in (1, 255, 256, 257, 3001):
        mesh = _edge_mesh(sk, n_vertices, seed=n_vertices)
        anim = lb.AnimationSystem(ctx, sk, clips, mesh, max_instances=max(counts))
        anim.setLaunch(skin_group=group)
        for n in counts:
            ci, tt = _times(n, clips, seed=n + n_vertices)
            anim.setInstances(ci, tt)
            anim.update(0.0, lb.PALETTE_MATRIX)
            anim.skin()
            assert anim.lastLaunch()[1] == g
            got = anim.getSkinned()
            mtx = anim.getMatrices()
            for i in range(n):
                exp = oracle.skin_vertices(mtx[i], mesh.positions, mesh.weights, mesh.indices)
                assert_bits_equal(got[i], exp, f"{bones} bones, group {group}, {n_vertices} vertices: instance {i} of {n}")
            assert anim.skinnedChecksum() == int(got.view(np.uint32).astype(np.uint64).sum())
        anim.close()


def test_set_launch_rejects_other_values(ctx):
    sk = scenes.skeleton(5)
    anim = lb.AnimationSystem(ctx, sk, _clips(sk), None, max_instances=4)
    assert anim.lastLaunch() == (0, 0)
    for lanes, group in ((2, 0), (64, 0), (-8, 0), (0, 32), (0, 2), (0, -4)):
        with pytest.raises(lb.LumixB200Error):
            anim.setLaunch(lanes, group)
    anim.close()
