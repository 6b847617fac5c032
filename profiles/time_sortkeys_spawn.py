"""Spawning k model instances per frame into the sort keys of the C2 scene (10 M entities, culling made device-authoritative by one in-place
set_many_device batch), k = 1 k, 10 k and 100 k; CUDA events around synchronised calls, median of REPS (default 5) after one untimed run:
  (a) device   add_many_device of the k new ids + spawn_instances_device of the same k + the next create_keys (+ radixSort);
  (b) host     what the sort keys take without a device spawn: set_instances of all entries (n + the ids spawned so far) of model_of / lod / flags / pose_frame
               (the fields a spawn writes) + set_transforms_device of as many transforms + the same create_keys.  The culling add of (b) is
               the same as (a)'s and is left out of its time.
Every repetition spawns k ids no repetition used before, so the scene grows by k per frame and nothing is removed.  Prints the card and
its power limit first."""
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes, sortkeys  # noqa: E402
from lumixengine_b200._lib import vp  # noqa: E402

KS = (1_000, 10_000, 100_000)


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
    ctx = lb.Context(0)
    scene = scenes.c2_scene()
    n = len(scene["entities"])
    reps = int(os.environ.get("REPS", "5"))
    cap = n + (reps + 1) * sum(KS)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    cs.set_replicas(1)
    still = np.arange(0, n, 1000, dtype=np.int32)
    d_still = [ctx.to_device(a) for a in (still, scene["pos"][still], scene["radius"][still])]
    cs.set_many_device(d_still[1], d_still[2], len(still), dev_entities=d_still[0], max_entity=n - 1)
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=23)
    S = lb.SortKeys(ctx, cap, sk["max_sort_key"] + 1, max_keys=1 << 22, max_instances=1 << 22)  # holds every spawn: no growth inside the timings
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    a = scenes.c2_frustum_args()
    view = sortkeys.make_view(a["position"], a["position"], 1.0 / 60.0, 1.0, 1, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
    rng = np.random.default_rng(5)
    # host arrays of all cap entries for (b): the scene's, then the new ids'
    model_all = np.concatenate([sk["model_of"], rng.integers(0, len(sk["models"]), cap - n).astype(np.uint32)])
    lod_all = np.concatenate([sk["lod"], np.zeros(cap - n, np.float32)])
    flags_all = np.concatenate([sk["flags"], np.zeros(cap - n, np.uint8)])
    pf_all = np.full(cap, 0xffffffff, np.uint32)
    tr_new = np.zeros(cap - n, lb.TRANSFORM_DTYPE)
    tr_new["pos"] = (rng.random((cap - n, 3)) * 2.0 - 1.0) * np.array([6000.0, 300.0, 6000.0])
    tr_new["rot"] = scenes.random_unit_quats(rng, cap - n)
    tr_new["scale"] = 1.0
    tr_all = np.empty(cap, lb.TRANSFORM_DTYPE)  # filled in place: np.concatenate would drop the 4 padding bytes of each 56-byte Transform
    tr_all[:n], tr_all[n:] = sk["transforms"], tr_new
    assert tr_all.dtype.itemsize == 56 and tr_all.nbytes == 56 * cap
    d_tr_all = ctx.to_device(tr_all)
    e0, e1, e2, e3 = ctx.event(), ctx.event(), ctx.event(), ctx.event()

    def keys():
        cs.cull_device(f, want_counts=False)
        S.createSortKeys(cs, view)

    rows = []
    top = n  # the next unused id
    for k in KS:
        add, spawn, keys_a, host, keys_b = [], [], [], [], []
        for r in range(reps + 1):
            ids = np.arange(top, top + k, dtype=np.int32)
            new = slice(top - n, top - n + k)
            rad = (0.5 + 4.5 * rng.random(k)).astype(np.float32)
            d = [ctx.to_device(x) for x in (ids, np.zeros(k, np.uint8), np.ascontiguousarray(tr_new["pos"][new]), rad, model_all[top:top + k],
                                            np.ascontiguousarray(tr_new[new]))]
            top += k
            ctx.synchronize(); ctx.record(e0)
            cs.add_many_device(d[2], d[3], d[1], k, dev_entities=d[0], max_entity=top - 1)
            ctx.record(e1)
            S.spawnInstancesDevice(d[0], d[4], d[5], k, top - 1)
            ctx.record(e2)
            keys()
            ctx.record(e3); ctx.synchronize()
            if r:
                add.append(ctx.elapsed_ms(e0, e1)); spawn.append(ctx.elapsed_ms(e1, e2)); keys_a.append(ctx.elapsed_ms(e2, e3))
            ctx.synchronize(); ctx.record(e0)
            S.setInstances(model_all[:top], lod_all[:top], flags_all[:top], pf_all[:top])
            S._err(S.L.lb200_sortkeys_set_transforms_device(S.h, vp(d_tr_all), C.c_uint32(top)))
            ctx.record(e1)
            keys()
            ctx.record(e2); ctx.synchronize()
            if r:
                host.append(ctx.elapsed_ms(e0, e1)); keys_b.append(ctx.elapsed_ms(e1, e2))
            for p in d:
                ctx.free_device(p)
        med = lambda x: float(np.median(x))  # noqa: E731
        row = dict(k=k, add_many_device_ms=med(add), spawn_instances_device_ms=med(spawn), create_keys_a_ms=med(keys_a),
                   device_total_ms=med(np.add(np.add(add, spawn), keys_a)), host_uploads_ms=med(host), create_keys_b_ms=med(keys_b),
                   host_total_ms=med(np.add(host, keys_b)))
        rows.append(row)
        print(f"k={k:>7}: (a) add {row['add_many_device_ms']:.3f} + spawn {row['spawn_instances_device_ms']:.3f} + keys {row['create_keys_a_ms']:.3f} = "
              f"{row['device_total_ms']:.3f} ms   (b) set_instances + set_transforms_device {row['host_uploads_ms']:.1f} + keys {row['create_keys_b_ms']:.3f} = "
              f"{row['host_total_ms']:.1f} ms")
    print(json.dumps(dict(card=name, power_limit=limit, entities=n, reps=reps, rows=rows)))
    ctx.free_device(d_tr_all)
    for p in d_still:
        ctx.free_device(p)
    S.close()
    cs.close()
    ctx.close()


if __name__ == "__main__":
    main()
