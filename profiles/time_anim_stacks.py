"""Sample lists (lb200_animation_set_samples) against clip mode + blend layers, at config 4's size (DESIGN.md §4.3).

  1. 100 k instances x 64 bones, DQ palette, stacks of 1, 2, 3 and 6 samples per instance: one update in sample-list mode against one
     update in clip mode with the same stack as base clip + 0, 1, 2 and 5 layers (both give the same bytes; checked before timing)
  2. update_many over 32 systems of 3125 instances, half in clip mode and half in sample-list mode (3-sample stacks, base clip + 2 layers
     on the clip-mode side), against the same systems all in clip mode
  3. --c4-only: clip-mode C4 alone (100 k instances x 64 bones, DQ palette, no layers), the figure that compares two builds of the library:
     run this script once per library (--lib PATH loads another liblumix_b200.so) and alternate the processes.
Device time: CUDA events around `calls` calls.  Forms alternate window by window, every shape is warmed up first, and the medians and
spreads of the windows are printed with the card, its power limit and its maximum SM clock, read in the same run.
Usage: python profiles/time_anim_stacks.py [--lib PATH] [--c4-only] [windows] [calls_per_window]"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lumixengine_b200 import _lib  # noqa: E402

args = sys.argv[1:]
if "--lib" in args:
    k = args.index("--lib")
    _lib.SO_PATH = os.path.abspath(args[k + 1])
    del args[k:k + 2]
C4_ONLY = "--c4-only" in args
args = [a for a in args if a != "--c4-only"]

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


def stack(n, clips, depth, seed):
    """depth entries per instance, clamped times below the clip length, the first at weight 1: clip mode's base clip + layers."""
    rng = np.random.default_rng(seed)
    lengths = np.array([c.length_ticks for c in clips])
    ci = rng.integers(0, len(clips), (n, depth)).astype(np.uint32)
    tt = (rng.random((n, depth)) * lengths[ci]).astype(np.uint32)
    w = rng.random((n, depth)).astype(np.float32)
    w[:, 0] = 1.0
    return ci, tt, w


def pair(ctx, sk, clips, n, depth, seed):
    """(sample-list system, clip-mode system) posing the same stacks; byte-equal outputs are checked."""
    ci, tt, w = stack(n, clips, depth, seed)
    lists = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    lists.setSamples(np.arange(0, n * depth + 1, depth, dtype=np.uint32), ci.reshape(-1), tt.reshape(-1), w.reshape(-1), np.zeros(n * depth, np.uint32))
    layered = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
    layered.setInstances(ci[:, 0], tt[:, 0])
    if depth > 1:
        layered.setLayers(ci[:, 1:], tt[:, 1:], w[:, 1:])
    lists.update(0.0, DQ)
    layered.update(0.0, DQ)
    assert lists.getDualQuats().tobytes() == layered.getDualQuats().tobytes(), f"depth {depth}: lists and layers differ"
    return lists, layered


def main():
    windows = int(args[0]) if len(args) > 0 else 9
    calls = int(args[1]) if len(args) > 1 else 20
    ctx = lb.Context(0)
    out = {"card": card(), "library": _lib.SO_PATH}
    sk = scenes.skeleton(BONES, seed=4)
    clips = [scenes.clip(sk, frames=30, seed=1), scenes.clip(sk, frames=45, seed=2)]
    if C4_ONLY:
        ci, tt = scenes.instance_times(N, clips)
        a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=N)
        a.setInstances(ci, tt)
        out["c4_clip_mode_update"] = timed(ctx, {"update": lambda: a.update(1.0 / 60.0, DQ)}, windows, calls)
        print(json.dumps(out))
        ctx.close()
        return
    for depth in (1, 2, 3, 6):
        lists, layered = pair(ctx, sk, clips, N, depth, seed=depth)
        out[f"1_stack_{depth}"] = timed(ctx, {"sample_lists": lambda: lists.update(0.0, DQ), f"clip_plus_{depth - 1}_layers": lambda: layered.update(0.0, DQ)},
                                        windows, calls)
        lists.close()
        layered.close()
    mixed, clip_only = [], []
    for s in range(32):
        lists, layered = pair(ctx, sk, clips, N // 32, 3, seed=100 + s)
        mixed.append(lists if s % 2 == 0 else layered)
        clip_only.append(layered)
    out["2_update_many_32_systems"] = timed(ctx, {"half_sample_lists": lambda: lb.AnimationSystem.updateMany(mixed, 0.0, DQ),
                                                  "all_clip_mode": lambda: lb.AnimationSystem.updateMany(clip_only, 0.0, DQ)}, windows, calls)
    print(json.dumps(out, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
