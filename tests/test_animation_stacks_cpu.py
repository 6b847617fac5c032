"""The restatement of an animator's blend-stack SAMPLE instructions (oracle_pose_stack) against reference-run vectors
(tests/golden/stack_kat.npz, made by tests/golden/make_stack_golden.py with the reference's own getPose / evalBlendStack), and the animator
binding (host/animators_b200.inl) compiled against the reference's headers with the engine's RenderModule."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from lumixengine_b200 import scenes
from oracle import build_ref, pystack
from bitexact import assert_bits_equal
from test_integration_compile import GXX, REF, ROOT, _copy_headers

BELOW = float(np.nextafter(np.float32(0.9999), np.float32(0)))


def stack_kat_inputs():
    """{bone count: (skeleton, clips, [(slot, weight, time_ticks, looped) per stack])}, from fixed seeds: stack lengths 0, 1, 2, 3 and 40,
    first samples below 0.9999, the weight edges and the time edges of looped and clamped samples."""
    out = {}
    for B in (1, 64, 196):
        sk = scenes.skeleton(64, seed=4) if B == 64 else scenes.skeleton(seed=B, parents=[-1] + [max(0, i - 1 - (i % 3)) for i in range(1, B)])
        clips = [scenes.clip(sk, frames=13, fps=30.0, seed=B, const_fraction=0.3),
                 scenes.clip(sk, frames=40, fps=24.0, seed=B + 1, pos_bits=(11, 14, 16), rot_bits=(12, 15, 16), const_fraction=0.3)]
        rng = np.random.default_rng(B)
        lengths = np.array([c.length_ticks for c in clips], np.int64)
        cases = []
        for k, n in enumerate([0, 1, 2, 3, 40, 1, 2, 3, 3, 40]):
            slot = rng.integers(0, len(clips), n).astype(np.uint32)
            L = lengths[slot]
            edge = rng.integers(0, 5, n)
            t = np.where(edge == 0, 0, np.where(edge == 1, L - 1, np.where(edge == 2, L, np.where(edge == 3, 2 * L + 17, (rng.random(n) * L).astype(np.int64)))))
            weight = np.array([0.0, BELOW, 0.9999, 1.0, 2.0, 0.3, 0.6], np.float32)[rng.integers(0, 7, n)]
            if n and k % 2:
                weight[0] = 0.4  # the first sample blends towards the bind pose
            cases.append((slot, weight, t.astype(np.uint32), rng.integers(0, 2, n).astype(np.uint32)))
        out[B] = (sk, clips, cases)
    return out


def test_oracle_pose_stack_equals_reference_vectors():
    kat = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stack_kat.npz"))
    n = 0
    for B, (sk, clips, cases) in stack_kat_inputs().items():
        for k, (slot, weight, time_ticks, looped) in enumerate(cases):
            pos, rot = pystack.pose_stack(sk, clips, slot, time_ticks, weight, looped)
            assert_bits_equal(pos, kat[f"b{B}_c{k}_pos"], f"B={B} stack {k}: positions")
            assert_bits_equal(rot, kat[f"b{B}_c{k}_rot"], f"B={B} stack {k}: rotations")
            n += 1
    assert n == len(kat.files) // 2


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "animation")), reason="reference tree not present")
def test_animator_binding_compiles_against_render_module():
    """host/animators_b200.inl instantiated with the engine's own RenderModule after controller.h, animation.h patched with
    host/animation_b200_decl.inl as INTEGRATION.md section 3 says."""
    host = os.path.join(ROOT, "lumixengine_b200", "host")
    with tempfile.TemporaryDirectory() as tmp:
        src = _copy_headers(tmp)
        patched = os.path.join(tmp, "patched")
        build_ref.patch_animation(src, patched)  # asserts the anchor of INTEGRATION.md section 3; controller.h beside the patched copy
        tu = os.path.join(tmp, "tu.cpp")
        open(tu, "w").write('#include "animation/animation.h"\n#include "animation/animation_module.h"\n#include "animation/controller.h"\n#include "core/log.h"\n'
                            '#include "core/stream.h"\n#include "renderer/model.h"\n#include "renderer/pose.h"\n#include "renderer/render_module.h"\n#include <string.h>\n'
                            '#include "animators_b200.inl"\nnamespace Lumix { template struct AnimatorsB200<RenderModule>; template struct AnimablesB200<RenderModule>; }\n')
        obj = os.path.join(tmp, "tu.o")
        cmd = GXX + ["-I", patched, "-I", src, "-I", os.path.join(REF, "external"), "-I", os.path.join(ROOT, "include"), "-I", host, tu, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "Lumix::AnimatorsB200<Lumix::RenderModule>::update(lb200_ctx*, Lumix::RenderModule&, Lumix::Span<Lumix::AnimatorB200Entry const>)" in syms
        for f in ("lb200_animation_create", "lb200_animation_set_samples", "lb200_animation_update_many", "lb200_animation_get_pose"):
            assert f in syms
