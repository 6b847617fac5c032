"""A topology change on config 3 (1 M nodes, depth 8, fan-out 7): one subtree re-parented per frame, host-synchronised time per frame
(medians over repetitions; every timed region ends in a device synchronise):
  (a) rebuild  destroy, create, set_locals, set_root_globals, propagate (what the engine binding did on every topology change);
  (b) device   set_parents, then propagate, on the same object;
and set_parents alone on the 1 M forest and on a depth-300 chain (40 nodes per level).  Asserts that (a) and (b) leave the same level
order and globals.  Prints the card and its power limit first.  Run from a tree whose library predates set_parents (the host-built level
order), it times (a) alone."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        name, limit = (s.strip() for s in out.strip().split(","))
        return name, limit
    except Exception:  # noqa: BLE001
        return "unknown", "unknown"


def reparented(parents, rng):
    """One subtree moved under a root of another tree (the root is never inside the subtree: roots have no parent)."""
    p = parents.copy()
    x = int(rng.choice(np.nonzero(p >= 0)[0]))
    roots = np.nonzero(p < 0)[0]
    top = x
    while p[top] >= 0:
        top = int(p[top])
    p[x] = int(rng.choice(roots[roots != top]))
    return p


def timed(ctx, fn):
    ctx.synchronize()
    t0 = time.perf_counter()
    fn()
    ctx.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    reps = int(os.environ.get("REPS", "9"))
    ctx = lb.Context(0)
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    rng = np.random.default_rng(5)
    frames = [reparented(parents, rng) for _ in range(reps + 1)]

    holder = {"h": lb.Hierarchy(ctx, parents)}

    def rebuild(p):
        holder["h"].close()
        h = lb.Hierarchy(ctx, p)
        h.setLocalTransforms(locals_)
        h.setRootTransforms(roots)
        h.propagate()
        holder["h"] = h

    if not hasattr(lb.Hierarchy, "setParents"):
        ta = [timed(ctx, lambda: rebuild(p)) for p in frames][1:]
        print(f"(a) destroy + create + locals + root globals + propagate: {np.median(ta):.3f} ms")
        print(json.dumps(dict(card=name, power_limit=limit, nodes=len(parents), reps=reps, rebuild_frame_ms=float(np.median(ta)))))
        return

    dev = lb.Hierarchy(ctx, parents)
    dev.setLocalTransforms(locals_)
    dev.setRootTransforms(roots)
    dev.propagate()

    def device(p):
        dev.setParents(p)
        dev.propagate()

    ta, tb = [], []
    for k, p in enumerate(frames):
        a, b = timed(ctx, lambda: rebuild(p)), timed(ctx, lambda: device(p))
        if k:  # the first frame grows the builder's scratch and the second topology set
            ta.append(a)
            tb.append(b)
        for x, y in zip(holder["h"].levelOrder(), dev.levelOrder()):
            assert np.array_equal(x, y), "rebuild and set_parents left different level orders"
        ga, gb = holder["h"].getTransforms(), dev.getTransforms()
        for f in ("pos", "rot", "scale"):
            assert ga[f].tobytes() == gb[f].tobytes(), "rebuild and set_parents left different globals"
    holder["h"].close()

    alone = {}
    chain = np.full(40 * 300, -1, np.int32)
    chain[40:] = np.arange(40 * 299, dtype=np.int32)  # node k + 40 under node k: 40 chains of depth 300
    for label, p in (("forest_1m", frames[-1]), ("chain_depth_300", chain)):
        h = lb.Hierarchy(ctx, p)
        h.setParents(p)
        ts = [timed(ctx, lambda: h.setParents(p)) for _ in range(reps)]
        alone[label] = dict(n=len(p), depth=h.depth, set_parents_ms=float(np.median(ts)))
        h.close()
    dev.close()

    row = dict(card=name, power_limit=limit, nodes=len(parents), reps=reps, rebuild_frame_ms=float(np.median(ta)),
               set_parents_frame_ms=float(np.median(tb)), set_parents_alone=alone)
    print(f"(a) destroy + create + locals + root globals + propagate: {row['rebuild_frame_ms']:.3f} ms")
    print(f"(b) set_parents + propagate:                             {row['set_parents_frame_ms']:.3f} ms")
    for label, r in alone.items():
        print(f"set_parents alone, {label} (n {r['n']}, depth {r['depth']}): {r['set_parents_ms']:.3f} ms")
    print(json.dumps(row))
    ctx.close()


if __name__ == "__main__":
    main()
