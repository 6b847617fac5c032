"""propagate_attached against propagate_moved on config 3 (1 M nodes): 1 k / 10 k / 100 k bone attachments to instances of one 100 k-instance
animation system, in 1 round (attached leaves following single roots) and in 3 rounds (chains leaf <- leaf <- leaf).  Both calls get the
same edits (1 % of the single roots moved) and no count read-back; every attachment is active (the system counts as posed).  Median of
alternating windows of CUDA-event time, ms per call.  Usage: python profiles/time_hierarchy_attached.py [windows] [calls_per_window]"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402


def main():
    windows = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    ctx = lb.Context(0)
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    n = len(parents)
    rng = np.random.default_rng(1)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    skel = scenes.skeleton(40)
    clips = [scenes.clip(skel, frames=30, seed=3)]
    anim = lb.AnimationSystem(ctx, skel, clips, None, max_instances=100_000)
    ci, tt = scenes.instance_times(100_000, clips)
    anim.setInstances(ci, tt)
    anim.update(1.0 / 60.0, lb.PALETTE_POSE)
    has_child = np.zeros(n, bool)
    has_child[parents[parents >= 0]] = True
    leaves = rng.permutation(np.nonzero(~has_child & (parents >= 0))[0])
    singles = np.nonzero((parents < 0) & ~has_child)[0]
    moved = rng.choice(singles, len(singles) // 100, replace=False).astype(np.uint32)
    vals = roots[moved].copy()
    results = []
    for k in (1_000, 10_000, 100_000):
        for rounds in (1, 3):
            att = leaves[:k]
            if rounds == 1:
                par = rng.choice(singles, k)
            else:  # chains of three: the second follows the first attached leaf, the third the second
                c = k // 3
                att = att[:3 * c]
                par = np.concatenate([rng.choice(singles, c), att[:c], att[c:2 * c]])
            m = len(att)
            rel = np.concatenate([rng.normal(size=(m, 3)).astype(np.float32), scenes.random_unit_quats(rng, m)], axis=1)
            h.setAttachments(att, par, np.zeros(m), rng.integers(0, 100_000, m), rng.integers(0, 40, m), rel)
            h.propagateAttached([anim])  # builds the rounds
            assert h.attachmentRounds()[1] == rounds
            ms = {"attached": [], "moved": []}
            e0, e1 = ctx.event(), ctx.event()
            for w in range(2 * windows):
                which = "attached" if w % 2 == 0 else "moved"
                total = 0.0
                for _ in range(calls):
                    h.setSubset(moved, vals, globals_=True)
                    ctx.record(e0)
                    if which == "attached":
                        h.propagateAttached([anim], read_count=False)
                    else:
                        h.propagateMoved(read_count=False)
                    ctx.record(e1)
                    ctx.synchronize()
                    total += ctx.elapsed_ms(e0, e1)
                ms[which].append(total / calls)
            r = {"nodes": n, "attachments": m, "rounds": rounds, "propagate_attached_ms": float(np.median(ms["attached"])),
                 "propagate_moved_ms": float(np.median(ms["moved"]))}
            results.append(r)
            print(json.dumps(r), flush=True)
    h.close()
    anim.close()
    ctx.close()


if __name__ == "__main__":
    main()
