"""IK instructions of animators' blend stacks, without a GPU: the restatement (oracle/oracle_ik.c: oracle_pose_stack_ik, oracle_eval_ik) against reference-run
vectors (tests/golden/ik_kat.npz, made by tests/golden/make_ik_golden.py with the reference's own evalBlendStack / evalIK over Models
that have a bone map), the IK arithmetic of csrc/lb200_math.cuh compiled for the host against the reference's own vec3ToVec3, nlerp,
inverted, length and conjugated, and the same stacks live against the reference harness where it was built.

ik_kat_inputs() is shared with tests/test_animation_ik_gpu.py and the golden generator.  Inputs where the reference computes a NaN (two
coincident joints) are outside the bit-for-bit contract and are not among them."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from lumixengine_b200 import scenes
from lumixengine_b200._lib import Clip
from lumixengine_b200.animation import Skeleton
from oracle import pyoracle as po
from oracle import pyik
from bitexact import assert_bits_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ik_kat.npz")
SHIM = po.ANIMATION_SHIM_SO
BELOW_0001 = float(np.nextafter(np.float32(0.001), np.float32(0)))  # the float just below 0.001f
ALPHAS = [0.0, BELOW_0001, 0.001, 0.5, 1.0]
CHAIN_LENGTHS = (1, 2, 3, 8, 32)


def axis_skeleton():
    """Bones along x (1, 2) and along y (3, 4) with identity rotations: 2-bone chains whose joints a target behind them turns by exactly
    180 degrees, the antiparallel branch of vec3ToVec3 with the direction along x (squaredLength(n) < 0.01) and along y."""
    parents = [-1, 0, 1, 0, 3]
    abs7 = np.zeros((5, 7), np.float32)
    abs7[:, 6] = 1
    abs7[1, 0], abs7[2, 0], abs7[3, 1], abs7[4, 1] = 1, 2, 1, 2
    return Skeleton(parents, abs7)


def ik_skeletons():
    """{name: skeleton}: 1, 64 and 196 bones, one with a 33-bone chain (and branches off it), the axis skeleton."""
    chain33 = [-1] + list(range(0, 32)) + [3, 10, 20, 33, 34, 30, 31]
    return {"b1": scenes.skeleton(seed=1, parents=[-1]), "b64": scenes.skeleton(64, seed=4),
            "b196": scenes.skeleton(seed=196, parents=[-1] + [max(0, i - 1 - (i % 3)) for i in range(1, 196)]),
            "c33": scenes.skeleton(seed=33, parents=chain33), "axis": axis_skeleton()}


def depths(parents):
    d = np.zeros(len(parents), np.int64)
    for i, p in enumerate(parents):
        d[i] = 0 if p < 0 else d[p] + 1
    return d


def chain_specs(sk):
    """(leaf, bone count) pairs: every length of CHAIN_LENGTHS the skeleton allows, with the first bone at the root and inside."""
    d = depths(sk.parents)
    out = []
    for n in CHAIN_LENGTHS:
        at_root = np.nonzero(d == n - 1)[0]
        inside = np.nonzero(d > n - 1)[0]
        if len(at_root):
            out.append((int(at_root[-1]), n))
        if len(inside):
            out.append((int(inside[len(inside) // 2]), n))
    return out


def _chain_root(sk, leaf, n):
    b = leaf
    for _ in range(n - 1):
        b = int(sk.parents[b])
    return b


def ik_kat_inputs():
    """{name: (skeleton, clips, [case])}, case = (slot, weight, time_ticks, looped, ik_after, ik_leaf, ik_bones, ik_alpha, ik_target [k, 3]).
    Per chain: IK on the bind pose, between samples, after the last sample, two ops at one position and the same chain twice; reachable
    and unreachable targets; alphas 0, the float below 0.001, 0.001, 0.5 and 1.  The axis skeleton adds both antiparallel sub-branches."""
    out = {}
    for si, (name, sk) in enumerate(ik_skeletons().items()):
        clips = [scenes.clip(sk, frames=13, fps=30.0, seed=si + 1, const_fraction=0.3),
                 scenes.clip(sk, frames=40, fps=24.0, seed=si + 2, pos_bits=(11, 14, 16), rot_bits=(12, 15, 16), const_fraction=0.3)]
        lengths = np.array([c.length_ticks for c in clips], np.int64)
        bind_abs = sk.bind_abs7[:, :3]
        rng = np.random.default_rng(100 + si)
        cases = []

        def samples(n):
            slot = rng.integers(0, len(clips), n).astype(np.uint32)
            t = (rng.random(n) * lengths[slot] * 1.5).astype(np.uint32)
            weight = np.array([1.0, 0.5, 0.25, 0.9999], np.float32)[rng.integers(0, 4, n)]
            return slot, weight, t, rng.integers(0, 2, n).astype(np.uint32)

        def target(leaf, n, reachable):
            root = bind_abs[_chain_root(sk, leaf, n)]
            reach = max(float(np.linalg.norm(bind_abs[leaf] - root)), 0.05) * max(1, n - 1)
            u = rng.normal(size=3)
            u /= np.linalg.norm(u)
            return (root + u * (0.4 * reach if reachable else 3.0 * reach + 1.0)).astype(np.float32)

        specs = chain_specs(sk) if name != "axis" else []
        for ci, (leaf, n) in enumerate(specs):
            for variant in range(5):
                ns = [0, 2, 3, 1, 2][variant]
                slot, weight, t, looped = samples(ns)
                after = {0: [0], 1: [1], 2: [3], 3: [1, 1], 4: [0, 2]}[variant]
                k = len(after)
                alpha = [ALPHAS[(ci + variant + j) % len(ALPHAS)] if variant else 1.0 for j in range(k)]
                if variant == 3:
                    alpha = [0.5, 1.0]
                tgt = np.stack([target(leaf, n, (variant + j + ci) % 2 == 0) for j in range(k)])
                cases.append((slot, weight, t, looped, np.array(after, np.uint32), np.full(k, leaf, np.uint32), np.full(k, n, np.uint32),
                              np.array(alpha, np.float32), tgt))
        if name == "axis":
            none = lambda: (np.zeros(0, np.uint32), np.zeros(0, np.float32), np.zeros(0, np.uint32), np.zeros(0, np.uint32))  # noqa: E731
            for leaf, tgt in ((2, (0.5, 0, 0)), (4, (0, 0.5, 0)), (2, (-5, 0, 0)), (4, (0, -5, 0))):
                for alpha in (1.0, 0.5):
                    cases.append((*none(), np.zeros(1, np.uint32), np.array([leaf], np.uint32), np.array([2], np.uint32), np.array([alpha], np.float32),
                                  np.array([tgt], np.float32)))
            # a 3-bone chain along x folded back over itself, a 1-bone chain, and two ops on both arms
            cases.append((*none(), np.zeros(1, np.uint32), np.array([2], np.uint32), np.array([3], np.uint32), np.ones(1, np.float32), np.array([[0.25, 0, 0]], np.float32)))
            cases.append((*none(), np.zeros(2, np.uint32), np.array([4, 2], np.uint32), np.array([1, 2], np.uint32), np.ones(2, np.float32),
                          np.array([[3, 1, 0], [0.5, 0, 0]], np.float32)))
        out[name] = (sk, clips, cases)
    return out


def expected(sk, clips, case):
    """The restatement's absolute pose for one case."""
    slot, weight, t, looped, after, leaf, bones, alpha, tgt = case
    return pyik.pose_stack_ik(sk, clips, slot, t, weight, looped, after, leaf, bones, alpha, tgt)


def test_oracle_pose_stack_ik_equals_reference_vectors():
    kat = np.load(GOLDEN)
    n = 0
    for name, (sk, clips, cases) in ik_kat_inputs().items():
        for k, case in enumerate(cases):
            pos, rot = expected(sk, clips, case)
            assert_bits_equal(pos, kat[f"{name}_c{k}_pos"], f"{name} case {k}: positions")
            assert_bits_equal(rot, kat[f"{name}_c{k}_rot"], f"{name} case {k}: rotations")
            n += 1
    assert n == len([f for f in kat.files if f.endswith("_pos") and "_c" in f])


def test_inputs_cover_the_edges():
    """What the vectors must contain: every chain length with its first bone at the root and inside, a 32-bone chain on the 33-bone
    chain, both antiparallel sub-branches, reachable and unreachable targets, every alpha, every position in the stack."""
    inputs = ik_kat_inputs()
    seen_len, seen_alpha, positions = set(), set(), set()
    for name, (sk, clips, cases) in inputs.items():
        d = depths(sk.parents)
        for slot, _, _, _, after, leaf, bones, alpha, _ in cases:
            for a, lf, b, al in zip(after, leaf, bones, alpha):
                seen_len.add((int(b), bool(d[lf] == b - 1)))
                seen_alpha.add(float(al))
                positions.add("first" if a == 0 else "last" if a == len(slot) else "between")
            if len(after) == 2 and after[0] == after[1]:
                positions.add("same position")
            if len(leaf) == 2 and leaf[0] == leaf[1] and bones[0] == bones[1]:
                positions.add("same chain twice")
    assert {(n, r) for n in CHAIN_LENGTHS for r in (True, False)} <= seen_len
    assert set(np.float32(ALPHAS).tolist()) <= seen_alpha
    assert {"first", "between", "last", "same position", "same chain twice"} <= positions


def test_no_nan_in_the_vectors():
    kat = np.load(GOLDEN)
    for f in kat.files:
        assert not np.isnan(kat[f]).any(), f


@pytest.fixture(scope="module")
def ik_math():
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "libik_math.so")
    # the flags the reference is built with: SSE2, no FMA contraction (scripts/genie.lua:339-342), as tests/test_host_math.py
    cmd = ["/usr/bin/g++", "-x", "c++", "-std=c++17", "-O2", "-msse2", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc,
           "-I", os.path.join(ROOT, "lumixengine_b200", "csrc"), os.path.join(ROOT, "tests", "host_math", "ik_math_harness.cpp"), "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def ik_math_inputs(n=1024, seed=7):
    """Random vectors and quaternions, plus the vec3ToVec3 edges: antiparallel pairs along x (squaredLength(n) < 0.01) and off the axes,
    pairs at cos just inside and outside (-1.0005, -0.9995), parallel pairs."""
    rng = np.random.default_rng(seed)
    v0 = rng.normal(size=(n, 3)).astype(np.float32)
    v1 = rng.normal(size=(n, 3)).astype(np.float32)
    m = n // 8
    v1[:m] = -v0[:m] * rng.uniform(0.1, 3, (m, 1)).astype(np.float32)                        # antiparallel, off the axes
    v0[m:2 * m] = np.array([1, 0, 0], np.float32) * rng.uniform(0.1, 3, (m, 1)).astype(np.float32)
    v0[m:2 * m, 1:] += rng.normal(scale=0.02, size=(m, 2)).astype(np.float32)                 # near x: squaredLength(n) < 0.01
    v1[m:2 * m] = -v0[m:2 * m]
    ang = rng.uniform(0.0, 0.08, m).astype(np.float32)                                        # cos near -1: both sides of the band
    v0[2 * m:3 * m] = np.stack([np.ones(m), np.zeros(m), np.zeros(m)], 1)
    v1[2 * m:3 * m] = np.stack([-np.cos(ang), np.sin(ang), np.zeros(m)], 1)
    v1[3 * m:4 * m] = v0[3 * m:4 * m] * np.float32(2)                                         # parallel
    qa = scenes.random_unit_quats(rng, n)
    qb = scenes.random_unit_quats(rng, n)
    t = rng.random(n).astype(np.float32)
    t[:8] = [0, 1, 0.5, 0.001, BELOW_0001, 0.25, 0.75, 0.9999]
    lrt = np.concatenate([rng.normal(size=(n, 3)).astype(np.float32), scenes.random_unit_quats(rng, n)], 1)
    return dict(v0=v0, v1=v1, qa=qa, qb=qb, t=t, lrt=np.ascontiguousarray(lrt, np.float32))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_ik_math_header_reproduces_reference_bits(ik_math):
    k = np.load(GOLDEN)
    n = len(k["m_v0"])
    c = np.ascontiguousarray
    o4, o7, o1 = np.zeros((n, 4), np.float32), np.zeros((n, 7), np.float32), np.zeros(n, np.float32)
    ik_math.ikm_vec3_to_vec3(_p(c(k["m_v0"])), _p(c(k["m_v1"])), _p(o4), C.c_uint(n))
    assert_bits_equal(o4, k["m_vec3_to_vec3"], "vec3ToVec3")
    ik_math.ikm_nlerp(_p(c(k["m_qa"])), _p(c(k["m_qb"])), _p(c(k["m_t"])), _p(o4), C.c_uint(n))
    assert_bits_equal(o4, k["m_nlerp"], "nlerp")
    ik_math.ikm_inverted(_p(c(k["m_lrt"])), _p(o7), C.c_uint(n))
    assert_bits_equal(o7, k["m_inverted"], "LocalRigidTransform::inverted")
    ik_math.ikm_length(_p(c(k["m_v0"])), _p(o1), C.c_uint(n))
    assert_bits_equal(o1, k["m_length"], "length")
    ik_math.ikm_conjugated(_p(c(k["m_qa"])), _p(o4), C.c_uint(n))
    assert_bits_equal(o4, k["m_conjugated"], "conjugated")
    # the vectors exercise both antiparallel sub-branches and the band's edges
    f = k["m_v0"] / np.linalg.norm(k["m_v0"], axis=1, keepdims=True)
    g = k["m_v1"] / np.linalg.norm(k["m_v1"], axis=1, keepdims=True)
    cos = (f * g).sum(1)
    anti = (cos > -1.0005) & (cos < -0.9995)
    small = f[:, 1] ** 2 + f[:, 2] ** 2 < 0.01
    assert (anti & small).sum() > 50 and (anti & ~small).sum() > 50 and ((cos < -0.99) & ~anti).sum() > 10


def run_ref_stack_ik(L, sk, clips, case):
    """One case through the reference harness (ref_pose_stack_ik): samples and IK instructions interleaved as `after` says."""
    slot, weight, t, looped, after, leaf, bones, alpha, tgt = case
    kind, cols = [], {k: [] for k in ("slot", "weight", "time", "looped", "leaf", "bones", "alpha", "target")}
    ik = 0
    for s in range(len(slot) + 1):
        while ik < len(after) and after[ik] == s:
            kind.append(2)
            for key, v in (("slot", 0), ("weight", 0), ("time", 0), ("looped", 0), ("leaf", leaf[ik]), ("bones", bones[ik]), ("alpha", alpha[ik])):
                cols[key].append(v)
            cols["target"].append(tgt[ik])
            ik += 1
        if s == len(slot):
            break
        kind.append(1)
        for key, v in (("slot", slot[s]), ("weight", weight[s]), ("time", t[s]), ("looped", looped[s]), ("leaf", 0), ("bones", 0), ("alpha", 0)):
            cols[key].append(v)
        cols["target"].append(np.zeros(3, np.float32))
    u = lambda k: np.array(cols[k], np.uint32)  # noqa: E731
    f = lambda k: np.array(cols[k], np.float32)  # noqa: E731
    B = sk.bone_count
    pos, rot = np.zeros((B, 3), np.float32), np.zeros((B, 4), np.float32)
    arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    rsk = po._skeleton_struct(sk, po.RefSkeleton)
    P = po._ptr
    assert L.ref_pose_stack_ik(C.byref(rsk), arr, C.c_uint32(len(clips)), P(np.array(kind, np.uint32)), P(u("slot")), P(f("weight")), P(u("time")), P(u("looped")),
                               P(u("leaf")), P(u("bones")), P(f("alpha")), P(np.ascontiguousarray(np.array(cols["target"], np.float32).reshape(-1, 3))),
                               C.c_uint32(len(kind)), P(pos), P(rot)) == 0
    return pos, rot


@pytest.mark.skipif(not os.path.exists(SHIM), reason="animator harness not built (no reference tree where build() ran)")
def test_restatement_equals_reference_live():
    L = C.CDLL(SHIM)
    for name, (sk, clips, cases) in ik_kat_inputs().items():
        for k, case in enumerate(cases):
            pos, rot = run_ref_stack_ik(L, sk, clips, case)
            ep, er = expected(sk, clips, case)
            assert_bits_equal(ep, pos, f"{name} case {k}: positions")
            assert_bits_equal(er, rot, f"{name} case {k}: rotations")
