"""The moved list of a propagate on config 3 (1 M nodes, depth 8, fan-out 7), device time from CUDA events, medians:
  (a) propagate against propagate_moved with 0 %, 1 %, 10 % and 100 % of the roots marked (mark_moved before each call, outside the window);
  (b) a frame of the device chain, today's against the moved list's:
      today: set_subset(roots) -> propagate -> refresh_spheres -> set_many_device(all n) -> cull
      moved: set_subset(roots) -> propagate_moved -> sortkeys_move_device(list) -> set_many_device(list) -> cull
      with 1 % of the roots moving each frame.
Each timed hierarchy is one of ROT rotated copies (the next call reads a hierarchy that is not resident in L2); the device is otherwise idle.
Checks first that both paths leave the same globals and visible set.  Prints the card and its power limit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return [s.strip() for s in out.strip().split(",")]
    except Exception:  # noqa: BLE001
        return ["unknown", "unknown", "unknown"]


def main():
    name, limit, clock = card()
    print(f"card: {name}, power limit {limit}, max SM clock {clock}")
    reps = int(os.environ.get("REPS", "15"))
    ROT = 3
    ctx = lb.Context(0)
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    n = len(parents)
    root_ids = np.nonzero(parents < 0)[0].astype(np.uint32)
    hs = []
    for _ in range(ROT):
        h = lb.Hierarchy(ctx, parents)
        h.setLocalTransforms(locals_)
        h.setRootTransforms(roots)
        h.propagate()
        hs.append(h)
    ev = [ctx.event() for _ in range(6)]
    rng = np.random.default_rng(5)

    def window(fn):
        ctx.synchronize()
        ctx.record(ev[0])
        fn()
        ctx.record(ev[1])
        ctx.synchronize()
        return ctx.elapsed_ms(ev[0], ev[1]) * 1e3

    # (a)
    a = {}
    for share in (0.0, 0.01, 0.10, 1.0):
        marked = rng.choice(root_ids, int(round(share * len(root_ids))), replace=False)
        tp, tm = [], []
        ks = set()
        for r in range(reps + 1):
            h = hs[r % ROT]
            t = window(h.propagate)
            h.markMoved(marked)
            holder = {}
            u = window(lambda: holder.setdefault("ml", h.propagateMoved(read_count=False)))
            ks.add(int(ctx.copy_to_host(holder["ml"].count_ptr, 1, np.uint32)[0]))
            if r:
                tp.append(t)
                tm.append(u)
        a[f"{share:.2f}"] = dict(marked_roots=len(marked), listed=sorted(ks), propagate_us=float(np.median(tp)), propagate_moved_us=float(np.median(tm)))
        print(f"(a) {100 * share:5.1f} % of the roots marked ({len(marked)} roots, {sorted(ks)} listed): propagate {a[f'{share:.2f}']['propagate_us']:.1f} us, "
              f"propagate_moved {a[f'{share:.2f}']['propagate_moved_us']:.1f} us")

    # (b)
    bounding = np.full(n, 1.0, np.float32)
    pos0, rad0 = hs[0].getSpheres(bounding)
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    systems = {}
    for path in ("today", "moved"):
        cs = lb.CullingSystem(ctx)
        cs.add(np.arange(n, dtype=np.int32), np.zeros(n, np.uint8), pos0, rad0)
        cs.flush()
        cs.set_replicas(1)
        S = lb.SortKeys(ctx, n, 64)
        S.setTransforms(np.zeros(n, lb.TRANSFORM_DTYPE))
        h = lb.Hierarchy(ctx, parents)
        h.setLocalTransforms(locals_)
        h.setRootTransforms(roots)
        h.propagate()
        h.refreshSpheres(bounding)
        h.markMoved([])
        h.propagateMoved(bounding)
        systems[path] = (cs, S, h)
    state = {"roots": roots.copy()}
    k_per_frame = max(1, len(root_ids) // 100)

    def frame_values():
        moved = rng.choice(root_ids, k_per_frame, replace=False).astype(np.uint32)
        vals = state["roots"][moved].copy()
        vals["pos"] += rng.normal(size=(len(moved), 3)) * 40.0
        state["roots"][moved] = vals
        return moved, vals

    def today(moved, vals):
        cs, S, h = systems["today"]
        ctx.record(ev[0])
        h.setSubset(moved, vals, globals_=True)
        h.propagate()
        d_pos, d_rad = h.refreshSpheres()
        ctx.record(ev[1])
        ch = cs.set_many_device(d_pos, d_rad, n)
        ctx.record(ev[2])
        cs.cull_device(f, want_counts=False)
        ctx.record(ev[3])
        ctx.synchronize()
        return [ctx.elapsed_ms(ev[i], ev[i + 1]) * 1e3 for i in range(3)], ch

    def moved_path(moved, vals):
        cs, S, h = systems["moved"]
        ctx.record(ev[0])
        h.setSubset(moved, vals, globals_=True)
        ml = h.propagateMoved()
        S.moveDevice(ml.entities, ml.transforms, ml.count)
        ctx.record(ev[1])
        ch = cs.set_many_device(ml.pos3, ml.radius, ml.count, dev_entities=ml.entities, max_entity=n - 1)
        ctx.record(ev[2])
        cs.cull_device(f, want_counts=False)
        ctx.record(ev[3])
        ctx.synchronize()
        S.endFrame()
        return [ctx.elapsed_ms(ev[i], ev[i + 1]) * 1e3 for i in range(3)], ch, ml.count

    bt, bm, ks = [], [], []
    for r in range(reps + 1):
        moved, vals = frame_values()
        ctx.synchronize()
        x, ch_t = today(moved, vals)
        y, ch_m, k = moved_path(moved, vals)
        assert ch_t == ch_m, "the two chains re-binned other movers"
        if r:
            bt.append(x)
            bm.append(y)
            ks.append(k)
    # both chains hold the same globals and cull the same entities
    ga, gb = systems["today"][2].getTransforms(), systems["moved"][2].getTransforms()
    for fld in ("pos", "rot", "scale"):
        assert ga[fld].tobytes() == gb[fld].tobytes()
    va, vb = systems["today"][0].cull(f), systems["moved"][0].cull(f)
    assert np.array_equal(np.sort(va.ids), np.sort(vb.ids))
    bt, bm = np.median(np.array(bt), axis=0), np.median(np.array(bm), axis=0)
    b = dict(moved_roots=k_per_frame, listed_median=int(np.median(ks)),
             today_us=dict(upload_propagate_spheres=float(bt[0]), set_many_device_all=float(bt[1]), cull=float(bt[2]), total=float(bt.sum())),
             moved_us=dict(upload_propagate_moved_move=float(bm[0]), set_many_device_list=float(bm[1]), cull=float(bm[2]), total=float(bm.sum())))
    print(f"(b) today: upload + propagate + refresh_spheres {bt[0]:.1f} us, set_many_device(all {n}) {bt[1]:.1f} us, cull {bt[2]:.1f} us, total {bt.sum():.1f} us")
    print(f"(b) moved: upload + propagate_moved + move_device {bm[0]:.1f} us, set_many_device({int(np.median(ks))} listed) {bm[1]:.1f} us, cull {bm[2]:.1f} us, "
          f"total {bm.sum():.1f} us")
    print(json.dumps(dict(card=name, power_limit=limit, max_sm_clock=clock, nodes=n, roots=len(root_ids), reps=reps, rotated=ROT, a=a, b=b)))
    for cs, S, h in systems.values():
        cs.close()
        S.close()
        h.close()
    for h in hs:
        h.close()
    ctx.close()


if __name__ == "__main__":
    main()
