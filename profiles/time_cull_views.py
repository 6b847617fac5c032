"""Device time of one frame's views on the C2 scene (10 M entities, the 8 replicas bench.py rotates through, so no timed cull re-reads an
L2-resident scene):
  (a) one cull_views call for all of the frame's views;
  (b) the same views as back-to-back cull_device(want_counts=False) calls on the context stream (programmatic launch overlaps them).
View sets: the main C2 view + the four shadow cascades prepareShadowCameras builds with the engine's default cascades (3, 10, 60, 150),
the same with cascades scaled to C2's far plane, and eight views (the default frame plus three more).  Each timed window holds ITERS frames
queued behind a sleep kernel, so the events measure the device alone; (a) and (b) alternate over RUNS windows, and the spread is printed.
Before timing, (a) and (b) are checked to give identical visible sets per view.  Prints the card and its power limit first."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402

REPLICAS = 8
LIGHT = (0.35, -0.85, 0.25)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        name, limit = (s.strip() for s in out.strip().split(","))
        return name, limit
    except Exception:  # noqa: BLE001
        return "unknown", "unknown"


def view_sets():
    a = scenes.c2_frustum_args()
    main = lb.frustum_perspective(**a)
    default = [main] + [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(a, LIGHT)]
    scaled = [main] + [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(a, LIGHT, tuple(c * a["far"] / 150.0 for c in scenes.DEFAULT_CASCADES))]
    more = [lb.frustum_perspective(**dict(a, position=(2000.0, 50.0, 1000.0), direction=(-0.7, -0.1, -0.7), far=1500.0)),   # a spot light
            lb.frustum_perspective(**dict(a, position=(-3000.0, 20.0, -2000.0), direction=(1.0, 0.0, 0.0), far=800.0)),    # another
            lb.frustum_perspective(**dict(a, direction=(0.0, 0.0, 1.0), far=2000.0))]                                     # a rear view
    return {"main + default cascades": default, "main + scaled cascades": scaled, "8 views": default + more}


def main():
    import torch
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    iters, runs = int(os.environ.get("ITERS", "20")), int(os.environ.get("RUNS", "7"))
    ctx = lb.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    scene = scenes.c2_scene()
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    cs.set_replicas(REPLICAS)
    e0, e1 = ctx.event(), ctx.event()

    def ids_of(ptr, r):
        """(type, id) keys of a device result, sorted: ids of type t at [type_offset[t], + type_count[t])."""
        keys = [ctx.copy_to_host(ptr + 4 * int(r.type_offset[t]), int(r.type_count[t]), np.uint32).astype(np.int64) + (t << 32) for t in range(256) if r.type_count[t]]
        return np.sort(np.concatenate(keys)) if keys else np.zeros(0, np.int64)

    def window(fn):
        """ITERS frames queued behind a ~10 ms sleep on the context stream: device time per frame in microseconds."""
        ctx.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)
        ctx.record(e0)
        for _ in range(iters):
            fn()
        ctx.record(e1)
        ctx.synchronize()
        return ctx.elapsed_ms(e0, e1) * 1e3 / iters

    rows = []
    for label, frusta in view_sets().items():
        # (a) and (b) agree view by view on the timed inputs
        out = cs.cull_views(frusta)
        fused = [ids_of(p, r) for p, r in out]
        visible = []
        for v, f in enumerate(frusta):
            p, r = cs.cull_device(f)
            assert int(r.total) == len(fused[v]) and np.array_equal(ids_of(p, r), fused[v]), (label, v)
            visible.append(int(r.total))
        cs.cull_views(frusta)
        views_bytes = cs.last_algorithmic_bytes()

        def a():
            cs.cull_views(frusta, want_counts=False)

        def b():
            for f in frusta:
                cs.cull_device(f, want_counts=False)

        a(); b()  # noqa: E702
        ta, tb = [], []
        for _ in range(runs):
            ta.append(window(a))
            tb.append(window(b))
        ll = cs.lastLaunch()
        a()
        la = cs.lastLaunch()
        row = dict(views=label, n_views=len(frusta), visible=visible, fused_us=float(np.median(ta)), fused_min_us=float(min(ta)), fused_max_us=float(max(ta)),
                   separate_us=float(np.median(tb)), separate_min_us=float(min(tb)), separate_max_us=float(max(tb)), fused_bytes=views_bytes,
                   fused_launch=la, separate_launch=ll)
        rows.append(row)
        print(f"{label:>24} ({len(frusta)} views, visible {visible}): (a) cull_views {row['fused_us']:.1f} us [{row['fused_min_us']:.1f}, {row['fused_max_us']:.1f}]   "
              f"(b) {len(frusta)} x cull_device {row['separate_us']:.1f} us [{row['separate_min_us']:.1f}, {row['separate_max_us']:.1f}]   "
              f"(a) launch {la['blocks']} blocks x chunk {la['chunk']}, {la['rounds']} rounds")
    print(json.dumps(dict(card=name, power_limit=limit, iters=iters, runs=runs, replicas=REPLICAS, rows=rows)))
    cs.close()
    ctx.close()


if __name__ == "__main__":
    main()
