"""Device time of the sort-key stage for all of a frame's views on the C2 scene (10 M entities, the sort-key setup of bench.py):
  (a) one create_keys_views call (with its sort) for every view of one cull_views;
  (b) the calls it replaces: select_view(v) + create_keys (with its sort) for v = 0, 1, ... on the context stream.
View sets: the main C2 view + the four shadow cascades prepareShadowCameras builds with the engine's default cascades, and the same with
cascades scaled to C2's far plane.  Every timed window starts from the same lod / Pose::frame state (reset through setInstances, untimed)
and holds one frame queued behind a sleep kernel, so the events measure the device alone; (a) and (b) alternate over RUNS windows, and the
median and spread are printed.  Before timing, (a) and (b) are checked to give the same outputs view by view.  Prints the card, its power
limit and its maximum SM clock first."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes, sortkeys as skm  # noqa: E402

LIGHT = (0.35, -0.85, 0.25)
FIELDS = ("keys", "values", "group_count", "group_offset", "group_renderables", "instance_data", "pose_list", "dirty_list")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout
        return tuple(s.strip() for s in out.strip().split(","))
    except Exception:  # noqa: BLE001
        return "unknown", "unknown", "unknown"


def canonical(out):
    """Outputs of one view in an order that does not depend on the launch: pairs and group members sorted."""
    o = np.lexsort((out["values"], out["keys"]))
    g = np.argsort(out["group_renderables"], kind="stable")
    return dict(keys=out["keys"][o], values=out["values"][o], group_count=out["group_count"], group_offset=out["group_offset"],
                group_renderables=out["group_renderables"][g], instance_data=out["instance_data"][g], pose_list=np.sort(out["pose_list"]),
                dirty_list=np.sort(out["dirty_list"]))


def main():
    import torch
    name, limit, clock = card()
    print(f"card: {name}, power limit {limit}, max SM clock {clock}")
    runs = int(os.environ.get("RUNS", "7"))
    ctx = lb.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    n = 10_000_000
    scene = scenes.c2_scene(n)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    cs.flush()
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=40)
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=1 << 23, max_instances=1 << 23)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    e0, e1 = ctx.event(), ctx.event()
    a = scenes.c2_frustum_args()
    sets = {"main + default cascades": [a] + scenes.shadow_cascade_args(a, LIGHT),
            "main + scaled cascades": [a] + scenes.shadow_cascade_args(a, LIGHT, tuple(c * a["far"] / 150.0 for c in scenes.DEFAULT_CASCADES))}

    def reset():
        S.setInstances(lod=sk["lod"], pose_frame=sk["pose_frame"])

    def window(fn):
        """One frame queued behind a ~10 ms sleep on the context stream: device time in microseconds."""
        reset()
        ctx.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)
        ctx.record(e0)
        fn()
        ctx.record(e1)
        ctx.synchronize()
        return ctx.elapsed_ms(e0, e1) * 1e3

    rows = []
    for label, args in sets.items():
        frusta = [lb.frustum_perspective(**args[0])] + [lb.frustum_ortho(**s) for s in args[1:]]
        views = [skm.make_view(s["position"], a["position"], 1.0 / 60.0, 1.0, 7, k > 0, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
                 for k, s in enumerate(args)]
        cs.cull_views(frusta, want_counts=False)

        def fused():
            S.createSortKeysViews(cs, views, sort=True, want_counts=False)

        def loop():
            for v, view in enumerate(views):
                cs.select_view(v)
                S.createSortKeys(cs, view, sort=True, want_counts=False)

        # (a) and (b) agree view by view on the timed inputs, state included
        reset()
        res = S.createSortKeysViews(cs, views)
        got = [canonical(S.readView(v, r)) for v, r in enumerate(res)]
        state_a = S.readView(0, res[0])
        reset()
        for v, view in enumerate(views):
            cs.select_view(v)
            r = S.createSortKeys(cs, view)
            assert (r.n_keys, r.n_instances, r.n_pose, r.n_dirty) == (res[v].n_keys, res[v].n_instances, res[v].n_pose, res[v].n_dirty), (label, v)
            exp = canonical(S.read(r))
            for f in FIELDS:
                assert np.array_equal(got[v][f], exp[f]), (label, v, f)
        state_b = S.read(r)
        assert np.array_equal(state_a["lod"].view(np.uint32), state_b["lod"].view(np.uint32)) and np.array_equal(state_a["pose_frame"], state_b["pose_frame"]), label
        fused(); loop()  # noqa: E702
        ta, tb = [], []
        for _ in range(runs):
            ta.append(window(fused))
            tb.append(window(loop))
        row = dict(views=label, n_views=len(views), n_keys=[int(r.n_keys) for r in res], n_instances=[int(r.n_instances) for r in res],
                   fused_us=float(np.median(ta)), fused_min_us=float(min(ta)), fused_max_us=float(max(ta)),
                   loop_us=float(np.median(tb)), loop_min_us=float(min(tb)), loop_max_us=float(max(tb)), launch=S.lastLaunch())
        rows.append(row)
        print(f"{label:>24} (keys {row['n_keys']}): (a) create_keys_views {row['fused_us']:.1f} us [{row['fused_min_us']:.1f}, {row['fused_max_us']:.1f}]   "
              f"(b) {len(views)} x select_view + create_keys {row['loop_us']:.1f} us [{row['loop_min_us']:.1f}, {row['loop_max_us']:.1f}]")
    print(json.dumps(dict(card=name, power_limit=limit, max_sm_clock=clock, runs=runs, rows=rows)))
    S.close()
    cs.close()
    ctx.close()


if __name__ == "__main__":
    main()
