"""The one-time cost of lb200_animation_set_root_motion (AnimationSystem.setRootMotion) when a group's system is built, and the per-frame
pose cost with and without root motion, which must not differ (the update runs the same kernels on the same tables).

Systems of 64 bones with 16, 64 and 256 clips of 60 or 600 frames (30 fps: 2 s / 20 s locomotion clips), every clip with root motion on
its root bone (a translation and a rotation track, all flags).  setRootMotion: host clock around the call, which returns after its kernels
(the root-motion tables, and the re-decode of clips that had root motion before) have run; the first call of a system and a repeated call
(which also decodes every clip again) are timed separately, median over `reps` systems.  Pose cost: CUDA events around `calls` updates of
10 k instances in clip mode, DQ palette, with and without root motion, alternating windows.  Prints the card, its power limit and its
maximum SM clock, read in the same run.
Usage: python profiles/time_anim_root_motion.py [reps] [windows] [calls_per_window]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402
from test_animation_root_motion_cpu import rm_clip  # noqa: E402

DQ = lb.PALETTE_DUAL_QUAT


def card():
    q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    return q.strip().splitlines()[0]


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    windows = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    calls = int(sys.argv[3]) if len(sys.argv) > 3 else 50
    ctx = lb.Context(0)
    sk = scenes.skeleton(64)
    out = {"card": card(), "set_root_motion_ms": {}, "update_us": {}}
    for frames in (60, 600):
        base = [rm_clip(sk, 0, "both", frames, (16, 16, 16), (15, 15, 15), seed=s) for s in range(8)]
        for n_clips in (16, 64, 256):
            clips = [base[c % len(base)] for c in range(n_clips)]
            tr = np.array([c.rootMotionTracks(0) for c in clips], np.int32)
            first, again = [], []
            for _ in range(reps):
                a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=1)
                ctx.synchronize()
                t0 = time.perf_counter()
                a.setRootMotion(np.full(n_clips, 7), tr[:, 0], tr[:, 1])
                first.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                a.setRootMotion(np.full(n_clips, 7), tr[:, 0], tr[:, 1])
                again.append(time.perf_counter() - t0)
                a.close()
            out["set_root_motion_ms"][f"{n_clips} clips x {frames + 1} frames"] = {"first": round(1e3 * float(np.median(first)), 3),
                                                                                   "repeated": round(1e3 * float(np.median(again)), 3)}
    # per-frame pose cost with and without root motion
    clips = [rm_clip(sk, 0, "both", 60, (16, 16, 16), (15, 15, 15), seed=s) for s in range(8)]
    tr = np.array([c.rootMotionTracks(0) for c in clips], np.int32)
    n = 10_000
    ci, tt = scenes.instance_times(n, clips)
    systems = {}
    for name in ("without", "with"):
        a = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
        a.setInstances(ci, tt)
        if name == "with":
            a.setRootMotion(np.full(len(clips), 7), tr[:, 0], tr[:, 1])
        systems[name] = a
    e0, e1 = ctx.event(), ctx.event()
    res = {k: [] for k in systems}
    for a in systems.values():
        for _ in range(3):
            a.update(0.0, DQ)
    ctx.synchronize()
    for w in range(windows):
        for name in (systems if w % 2 == 0 else reversed(list(systems))):
            a = systems[name]
            ctx.synchronize()
            ctx.record(e0)
            for _ in range(calls):
                a.update(0.0, DQ)
            ctx.record(e1)
            ctx.synchronize()
            res[name].append(1e3 * ctx.elapsed_ms(e0, e1) / calls)
    for name, v in res.items():
        out["update_us"][name] = {"median": round(float(np.median(v)), 2), "min": round(float(np.min(v)), 2), "max": round(float(np.max(v)), 2)}
    for a in systems.values():
        a.close()
    ctx.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
