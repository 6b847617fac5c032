"""Skinning palettes of the instances createSortKeys claims (lb200_sortkeys_build_palettes, DESIGN.md §4.7).

Scene: a C2-like culling scene (1 M entities over 6000 x 300 x 6000 m, the C2 camera) in which 100 k of the visible meshes are skinned
instances of one skinned model, posed by four animation systems of 64 (config 4's skeleton), 32, 17 and 100 bones with 40 k, 30 k,
20 k and 10 k instances.  The drawn fraction f is set through Pose::frame: the instances outside it already carry this frame's number, so
createSortKeys claims f of the 100 k and the pose list holds them.
  1. build_palettes alone at f = 5, 20, 50, 100 %: device time, and the least time the algorithmic bytes (28 B pose read + 32 B palette
     write per listed bone) take at the data sheet's 3.35 TB/s, as a share of it
  2. one update_many with DUAL_QUAT | POSE against update_many with POSE + build_palettes at the same fractions
Device time: CUDA events around `calls` calls; the forms of (2) alternate window by window, every shape is warmed up first, and the
medians (and min / max) of the windows are printed with the card, its power limit and its maximum SM clock, read in the same run.  Each
fraction's build is checked against the dual quaternions of the DUAL_QUAT update first.
Usage: python profiles/time_sortkeys_palettes.py [windows] [calls_per_window] [out.json]"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes, sortkeys  # noqa: E402

DQ, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_POSE
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SYSTEMS = ((64, 40_000), (32, 30_000), (17, 20_000), (100, 10_000))
FRACTIONS = (0.05, 0.2, 0.5, 1.0)
FRAME = 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def timed(ctx, fn, calls):
    a, b = ctx.event(), ctx.event()
    ctx.record(a)
    for _ in range(calls):
        fn()
    ctx.record(b)
    ctx.synchronize()
    return 1000.0 * ctx.elapsed_ms(a, b) / calls  # us per call


def main():
    windows = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    out_path = sys.argv[3] if len(sys.argv) > 3 else None
    ctx = lb.Context(0)
    n = 1_000_000
    sc = scenes.cull_scene(n, (6000.0, 300.0, 6000.0), seed=2)
    sk = scenes.sortkey_setup(n, sc["types"], sc["pos"], seed=8, skinned_fraction=0.0)  # model 0 alone is skinned
    sk["models"]["lod_distances"][0] = np.finfo(np.float32).max  # drawn at any distance
    cs = lb.CullingSystem(ctx)
    cs.add(sc["entities"], sc["types"], sc["pos"], sc["radius"])
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    visible = np.asarray(cs.cull(f).ids, np.int64)
    rng = np.random.default_rng(3)
    total = sum(k for _, k in SYSTEMS)
    skinned = rng.permutation(visible)[:total].astype(np.int32)
    assert len(skinned) == total, f"{len(visible)} visible entities, {total} wanted"
    model_of = sk["model_of"].copy()
    model_of[model_of == 0] = 1
    model_of[skinned] = 0
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * len(visible), max_instances=4 * len(visible))
    S.setModels(sk["models"], sk["meshes"])
    lod = sk["lod"].copy()
    lod[skinned] = 0.0  # settled on LOD 0, which holds the skinned meshes
    S.setInstances(model_of, lod, np.zeros(n, np.uint8), sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    systems, at = [], 0
    for bones, k in SYSTEMS:
        skel = scenes.skeleton(bones, seed=bones)
        clips = [scenes.clip(skel, frames=60, fps=30.0, seed=bones + 1), scenes.clip(skel, frames=45, fps=24.0, seed=bones + 2)]
        a = lb.AnimationSystem(ctx, skel, clips, max_instances=k)
        a.setInstances(*scenes.instance_times(k, clips, seed=bones + 3))
        a.setEntities(skinned[at:at + k])
        systems.append(a)
        at += k
    view = sortkeys.make_view(scenes.c2_frustum_args()["position"], scenes.c2_frustum_args()["position"], 0.0, 1.0, FRAME, False, sk["max_sort_key"],
                              sk["layer_to_bucket"], sk["depth_sorted_buckets"])
    bones_of = np.zeros(n, np.int64)
    for (bones, k), i in zip(SYSTEMS, np.cumsum([0] + [k for _, k in SYSTEMS])[:-1]):
        bones_of[skinned[i:i + k]] = bones
    rows = []
    hw = card()
    print("card, power limit, max SM clock:", hw)
    for frac in FRACTIONS:
        drawn = rng.permutation(skinned)[:int(round(frac * total))]
        pf = np.full(n, FRAME, np.uint32)
        pf[drawn] = 0xffffffff
        S.setInstances(pose_frame=pf)
        cs.cull_device(f, want_counts=False)
        res = S.createSortKeys(cs, view, sort=False)
        listed = S.read(res)["pose_list"]
        assert len(listed) == len(drawn), (len(listed), len(drawn))
        # correctness first: the build against the DUAL_QUAT update of the same poses
        lb.AnimationSystem.updateMany(systems, 0.0, DQ | POSE)
        S.buildPalettes(systems)
        pal = S.readPalettes()
        for s, a in enumerate(systems):
            ents = skinned[sum(k for _, k in SYSTEMS[:s]):sum(k for _, k in SYSTEMS[:s + 1])]
            sel = np.nonzero(np.isin(ents, listed))[0][:200]
            exp = a.getDualQuats()
            for i in sel:
                o = int(pal["offset"][ents[i]])
                assert np.array_equal(pal["dual_quats"][o:o + a.skeleton.bone_count].view(np.uint32), exp[i].view(np.uint32))
        listed_bones = int(bones_of[listed].sum())
        assert pal["n_bones"] == listed_bones
        build = lambda: S.buildPalettes(systems)  # noqa: E731
        upd_dq = lambda: lb.AnimationSystem.updateMany(systems, 0.0, DQ | POSE)  # noqa: E731

        def upd_build():
            lb.AnimationSystem.updateMany(systems, 0.0, POSE)
            S.buildPalettes(systems)
        for fn in (build, upd_dq, upd_build):
            timed(ctx, fn, calls)
        t = {"build": [], "update_dq_pose": [], "update_pose_build": []}
        for _ in range(windows):
            t["build"].append(timed(ctx, build, calls))
            t["update_dq_pose"].append(timed(ctx, upd_dq, calls))
            t["update_pose_build"].append(timed(ctx, upd_build, calls))
        med = {k: float(np.median(v)) for k, v in t.items()}
        algo = listed_bones * 60
        row = dict(fraction=frac, listed=int(len(listed)), listed_bones=listed_bones, algorithmic_bytes=algo,
                   build_us=med["build"], build_min_max=[min(t["build"]), max(t["build"])],
                   build_hbm_share=algo / HBM_BYTES_PER_S / (med["build"] * 1e-6),
                   update_dq_pose_us=med["update_dq_pose"], update_pose_plus_build_us=med["update_pose_build"],
                   spread_dq_pose=[min(t["update_dq_pose"]), max(t["update_dq_pose"])], spread_pose_build=[min(t["update_pose_build"]), max(t["update_pose_build"])])
        rows.append(row)
        print(json.dumps(row))
    print("| drawn | listed bones | build_palettes (us) | share of 3.35 TB/s | update_many DQ+POSE (us) | update_many POSE + build (us) |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['fraction'] * 100:.0f} % | {r['listed_bones']:,} | {r['build_us']:.1f} | {100 * r['build_hbm_share']:.0f} % | {r['update_dq_pose_us']:.1f} | {r['update_pose_plus_build_us']:.1f} |")
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        json.dump(dict(card=hw, windows=windows, calls=calls, rows=rows), open(out_path, "w"), indent=1)
    for a in systems:
        a.close()
    S.close()
    ctx.close()


if __name__ == "__main__":
    main()
