"""Spawn / despawn batches on the C2 scene (10 M entities) made device-authoritative by one set_many_device batch; CUDA-event time per batch
(events around each synchronised call, so host work inside a call counts) for k = 1 k, 10 k and 100 k new entities:
  (a) device   add_many_device of k entities + remove_many_device of the same k;
  (b) host     the same edits through add_many / remove_many (the first host edit pulls the device state back) + the next cull, with the
               device made authoritative again (one in-place set_many_device, untimed) before every repetition.
The cull alone is timed as well, so (b) can be read against (a) + one cull.  Prints the card and its power limit first."""
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


def main():
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    reps = int(os.environ.get("REPS", "5"))
    ctx = lb.Context(0)
    scene = scenes.c2_scene()
    n = len(scene["entities"])
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    cs.cull_device(f, want_counts=False)
    still = np.arange(0, n, 1000, dtype=np.int32)  # in-place movers: one batch that makes the device authoritative and changes nothing
    d_still = [ctx.to_device(a) for a in (still, scene["pos"][still], scene["radius"][still])]

    def authoritative():
        cs.set_many_device(d_still[1], d_still[2], len(still), dev_entities=d_still[0], max_entity=n - 1)

    authoritative()
    e0, e1, e2 = ctx.event(), ctx.event(), ctx.event()

    def cull_ms():
        ts = []
        for _ in range(reps + 1):
            ctx.synchronize(); ctx.record(e0)
            cs.cull_device(f, want_counts=False)
            ctx.record(e1); ctx.synchronize()
            ts.append(ctx.elapsed_ms(e0, e1))
        return float(np.median(ts[1:]))

    rng = np.random.default_rng(7)
    rows = []
    for k in (1_000, 10_000, 100_000):
        ids = np.arange(n, n + k, dtype=np.int32)
        types = rng.choice(np.array([0, 1, 2, 3], np.uint8), k, p=[0.85, 0.05, 0.05, 0.05]).astype(np.uint8)
        pos = (rng.random((k, 3)) * 2.0 - 1.0) * np.array([6000.0, 300.0, 6000.0])
        rad = (0.5 + 4.5 * rng.random(k)).astype(np.float32)
        d = [ctx.to_device(a) for a in (ids, types, pos, rad)]
        add, rem = [], []
        for r in range(reps + 1):  # the first repetition grows the buffers and is not counted
            ctx.synchronize(); ctx.record(e0)
            cs.add_many_device(d[2], d[3], d[1], k, dev_entities=d[0], max_entity=n + k - 1)
            ctx.record(e1)
            cs.remove_many_device(d[0], k)
            ctx.record(e2); ctx.synchronize()
            if r:
                add.append(ctx.elapsed_ms(e0, e1)); rem.append(ctx.elapsed_ms(e1, e2))
        for p in d:
            ctx.free_device(p)
        assert cs.entity_count() == n
        host, wall = [], []
        for r in range(reps + 1):
            authoritative()
            ctx.synchronize(); ctx.record(e0)
            t0 = time.perf_counter()
            cs.add(ids, types, pos, rad)
            cs.remove(ids)
            cs.cull_device(f, want_counts=False)
            ctx.record(e1); ctx.synchronize()
            t1 = time.perf_counter()
            if r:
                host.append(ctx.elapsed_ms(e0, e1)); wall.append((t1 - t0) * 1e3)
        assert cs.entity_count() == n
        authoritative()
        row = dict(k=k, device_add_ms=float(np.median(add)), device_remove_ms=float(np.median(rem)), device_ms=float(np.median(np.add(add, rem))),
                   host_route_ms=float(np.median(host)), host_route_wall_ms=float(np.median(wall)))
        rows.append(row)
        print(f"k={k:>7}: (a) device add {row['device_add_ms']:.3f} ms + remove {row['device_remove_ms']:.3f} ms = {row['device_ms']:.3f} ms   "
              f"(b) host add + remove + cull {row['host_route_ms']:.1f} ms (wall {row['host_route_wall_ms']:.1f} ms)")
    c = cull_ms()
    print(f"one C2 cull alone: {c:.3f} ms")
    print(json.dumps(dict(card=name, power_limit=limit, entities=n, reps=reps, cull_ms=c, rows=rows)))
    for p in d_still:
        ctx.free_device(p)
    cs.close()
    ctx.close()


if __name__ == "__main__":
    main()
