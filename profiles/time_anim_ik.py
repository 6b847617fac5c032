"""IK instructions in blend stacks (lb200_animation_set_stacks) against the same stacks without them, at config 4's size (DESIGN.md §4.3).

100 k instances x 64 bones (a 40-bone chain with branches, so that a 32-bone chain fits), DQ palette, every instance a stack of 2 samples:
  - 2 samples (set_samples: the kernel without IK)
  - 2 samples + one 3-bone IK op after them
  - 2 samples + one 32-bone IK op after them
Targets are reachable for half of the instances and unreachable for the other half; alpha 0.5.  Device time: CUDA events around `calls`
updates.  Forms alternate window by window, every form is warmed up first, and the medians and spreads of the windows are printed with the
card, its power limit and its maximum SM clock, read in the same run.
Usage: python profiles/time_anim_ik.py [windows] [calls_per_window]"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402

DQ = lb.PALETTE_DUAL_QUAT
N, BONES = 100_000, 64


def card():
    q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    return q.strip().splitlines()[0]


def timed(ctx, forms, windows, calls):
    """forms: name -> callable of one frame.  Alternating windows; per form the median (and min..max) device ms per call."""
    e0, e1 = ctx.event(), ctx.event()
    res = {k: [] for k in forms}
    for f in forms.values():
        for _ in range(3):
            f()
    ctx.synchronize()
    for w in range(windows):
        for name, f in (forms.items() if w % 2 == 0 else reversed(list(forms.items()))):
            ctx.synchronize()
            ctx.record(e0)
            for _ in range(calls):
                f()
            ctx.record(e1)
            ctx.synchronize()
            res[name].append(ctx.elapsed_ms(e0, e1) / calls)
    return {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))} for k, v in res.items()}


def main():
    windows = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    ctx = lb.Context(0)
    out = {"card": card()}
    parents = [-1] + [i - 1 for i in range(1, 40)] + [i - 4 for i in range(40, BONES)]
    sk = scenes.skeleton(seed=4, parents=parents)
    clips = [scenes.clip(sk, frames=30, seed=1), scenes.clip(sk, frames=45, seed=2)]
    rng = np.random.default_rng(3)
    lengths = np.array([c.length_ticks for c in clips])
    ci = rng.integers(0, len(clips), 2 * N).astype(np.uint32)
    tt = (rng.random(2 * N) * lengths[ci]).astype(np.uint32)
    w = np.tile(np.array([1.0, 0.5], np.float32), N)
    lo = np.zeros(2 * N, np.uint32)
    offsets = np.arange(0, 2 * N + 1, 2, dtype=np.uint32)
    systems = {}
    a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=N)
    a.setSamples(offsets, ci, tt, w, lo)
    systems["2_samples"] = a
    root = sk.bind_abs7[0, :3]
    for n_bones in (3, 32):
        leaf = 39  # depth 39: a 32-bone chain starts inside the skeleton
        far = np.where(np.arange(N)[:, None] % 2 == 0, 0.5, 50.0)
        target = (root + far * rng.normal(size=(N, 3))).astype(np.float32)
        s = lb.AnimationSystem(ctx, sk, clips, None, max_instances=N)
        s.setStacks(offsets, ci, tt, w, lo, np.arange(N + 1, dtype=np.uint32), np.full(N, 2, np.uint32), np.full(N, leaf, np.uint32),
                    np.full(N, n_bones, np.uint32), np.full(N, 0.5, np.float32), target)
        systems[f"2_samples_ik_{n_bones}_bones"] = s
    out["100k_x_64_dq"] = timed(ctx, {k: (lambda s=s: s.update(0.0, DQ)) for k, s in systems.items()}, windows, calls)
    print(json.dumps(out, indent=1))
    for s in systems.values():
        s.close()
    ctx.close()


if __name__ == "__main__":
    main()
