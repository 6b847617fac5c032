"""fillClusters on the device (lb200_clusters_fill, DESIGN.md §4.8) against the reference's own host code on one core.

Scene: C2 (10 M entities, 5 % LOCAL_LIGHT) with cull radius = range, 20 % of the lights casting shadows, 37 atlas entries, 16 env and 16
refl probes; its main view (the C2 camera) culled once with cull_device, then
  1. fill at 1920 x 1080 and 3840 x 2160: the call as the caller sees it (host clock around back-to-back calls; each ends in its
     read-back and synchronisation, so this is the end-to-end time, launches and host work included), medians over windows, with the
     lights, map entries and the algorithmic bytes of DESIGN.md §4.8 over that time as a share of the data sheet's 3.35 TB/s;
  2. the reference's fillClusters code (oracle/_ref/libclusters_shim_b200.so: the light loop with AtlasSorter, the planes, the count,
     offset and map passes) on the same light order, on one core, timed with the host clock: one call per sample, its inputs converted
     and its outputs allocated (map[] with room for every entry) before the clock starts;
  3. at 1920 x 1080 again, the AtlasSorter pass at its worst: every visible light casts shadows and the priorities rise along the light
     order (fov set so that fov * range^3 / distance is the light's position in the order), so that the screen of
     clusters_atlas_kernel lets every light through to warp 0's serial push.
Each row's device output (lights, clusters, map, the AtlasSorter list, the uncast lights with an atlas entry, and light_entities as a
permutation of the cull's LOCAL_LIGHT segment) is checked against that code first.  Prints the card, its power limit and its maximum SM
clock.
Usage: python profiles/time_clusters.py [windows] [calls_per_window] [out.json]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import clusters as lc  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402
from oracle import pyclusters as pc  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
RESOLUTIONS = ((1920, 1080), (3840, 2160))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def algorithmic_bytes(n_lights, n_probes, n_map, n_clusters):
    """Per light: id 4 + entity record 64 + PointLight 32 + atlas entry 4 read, ClusterLight 64 + entity 4 + priority 4 + flags 1 + ranges
    8 written, priority + flags + entity read again by the atlas pass (9); per probe 16 read + 8 written; per map entry: the pair written
    (16), read and written by each of the two sort passes (64), read by the table pass (8 of the value) and the map written (4); per
    cluster 16 written (its binary searches stay in L2)."""
    return n_lights * (104 + 81 + 9) + n_probes * 24 + n_map * (16 + 64 + 8 + 4) + n_clusters * 16


def main():
    windows = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    out_path = sys.argv[3] if len(sys.argv) > 3 else None
    shim = pc.load("shim")
    if shim is None:
        sys.exit("oracle/_ref/libclusters_shim_b200.so is not built: run build() where the reference sources are")
    sc = scenes.c2_scene()
    n = len(sc["entities"])
    rng = np.random.default_rng(11)
    ctx = lb.Context(0)
    cs = lb.CullingSystem(ctx)
    cs.add(sc["entities"], sc["types"], sc["pos"], sc["radius"])
    tr = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr["pos"] = sc["pos"]
    tr["rot"] = (0.0, 0.0, 0.0, 1.0)
    tr["scale"] = 1.0
    sk = lb.SortKeys(ctx, n, 1, max_keys=1024, max_instances=1024)
    sk.setTransforms(tr)
    cl = lb.Clusters(ctx, n)
    lights = np.flatnonzero(sc["types"] == 2).astype(np.int32)
    pl = np.zeros(n, lc.POINT_LIGHT_DTYPE)
    m = len(lights)
    pl["color"][lights] = rng.uniform(0, 1, (m, 3))
    pl["intensity"][lights] = rng.uniform(0, 10, m)
    pl["fov"][lights] = rng.uniform(0.1, 3.0, m)
    pl["attenuation_param"][lights] = rng.uniform(0, 100, m)
    pl["range"][lights] = sc["radius"][lights]
    pl["flags"][lights] = (rng.random(m) < 0.2).astype(np.uint32)
    cl.setPointLights(lights, pl[lights])
    atlas = np.full(n, -1, np.int32)
    with_entry = rng.choice(lights, 37, replace=False).astype(np.int32)
    atlas[with_entry] = np.arange(37)
    cl.setAtlas(with_entry, atlas[with_entry])
    env = np.zeros(16, lc.CLUSTER_ENV_PROBE_DTYPE)
    env["pos"] = rng.uniform(-2000, 2000, (16, 3))
    env["outer_range"] = rng.uniform(1, 40, (16, 3))
    refl = np.zeros(16, lc.CLUSTER_REFL_PROBE_DTYPE)
    refl["pos"] = rng.uniform(-2000, 2000, (16, 3))
    refl["half_extents"] = rng.uniform(1, 40, (16, 3))
    a = scenes.c2_frustum_args()
    rows = []
    for w, h, order in [(w, h, "cull") for w, h in RESOLUTIONS] + [(1920, 1080, "rising priorities")]:
        f = lb.frustum_perspective(a["position"], a["direction"], a["up"], a["fov"], w / h, a["near"], a["far"])
        dev, cres = cs.cull_device(f)
        off, cnt = cres.type_offset[2], cres.type_count[2]
        visible = ctx.copy_to_host(dev, off + cnt, np.uint32)[off:]
        view = lc.make_view(a["position"], f, w, h)
        if order != "cull":
            # the light order of this cull, then fov so that light k's priority is about k + 1
            ents = cl.read(cl.fillClusters(sk, cs, view, env, refl))["light_entities"]
            d = np.sqrt(((tr["pos"][ents] - np.asarray(a["position"])) ** 2).sum(1))
            r3 = pl["range"][ents].astype(np.float64) ** 3
            pl["fov"][ents] = (np.arange(1, len(ents) + 1) * d / r3).astype(np.float32)
            pl["flags"][ents] |= lc.CAST_SHADOWS
            cl.setPointLights(ents, pl[ents])
        res = cl.fillClusters(sk, cs, view, env, refl)
        got = cl.read(res)
        ents = got["light_entities"]
        assert np.array_equal(np.sort(ents), np.sort(visible.astype(np.int32))), "light_entities is not the cull's LOCAL_LIGHT segment"
        pts = np.array([[f.points[i][c] for c in range(3)] for i in range(8)], np.float32).reshape(24)
        args = (pts, w, h, a["position"], ents, tr["pos"][ents], tr["rot"][ents], pl[ents], atlas[ents], env, refl)
        exp = pc.fill(*args, which="shim")
        assert np.array_equal(got["lights"].view(np.uint8), exp["lights"].view(np.uint8)) and np.array_equal(got["map"], exp["map"])
        assert np.array_equal(got["clusters"].view(np.uint8), exp["clusters"].view(np.uint8))
        assert np.array_equal(lc.shadow_list(res).view(np.uint8), exp["shadow"].view(np.uint8))
        assert np.array_equal(np.array(res.uncast[:res.n_uncast], np.int32), exp["uncast"])
        for _ in range(3):
            cl.fillClusters(sk, cs, view, env, refl)
        wall = []
        for _ in range(windows):
            ctx.synchronize()
            t0 = time.perf_counter()
            for _ in range(calls):
                cl.fillClusters(sk, cs, view, env, refl)
            wall.append((time.perf_counter() - t0) / calls * 1e6)
        call, _ = pc.prepare(*args, which="shim", map_cap=len(exp["map"]))
        host = []
        for _ in range(5):
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e6)
        nbytes = algorithmic_bytes(res.n_lights, 32, res.n_map, res.n_clusters)
        row = dict(w=w, h=h, light_order=order, n_casters=int((pl["flags"][ents] & lc.CAST_SHADOWS).astype(bool).sum()), n_lights=int(res.n_lights), n_map=int(res.n_map), n_clusters=int(res.n_clusters), n_shadow=int(res.n_shadow),
                   fill_call_us=float(np.median(wall)), fill_call_us_min=float(np.min(wall)), fill_call_us_max=float(np.max(wall)),
                   algorithmic_bytes=int(nbytes), hbm_share_of_call_time=nbytes / HBM_BYTES_PER_S / (np.median(wall) * 1e-6),
                   reference_one_core_us=float(np.median(host)), reference_one_core_us_min=float(np.min(host)))
        rows.append(row)
        print(json.dumps(row))
    rec = dict(card=card(), windows=windows, calls=calls, rows=rows)
    print(json.dumps(dict(card=rec["card"])))
    if out_path:
        with open(out_path, "w") as fh:
            json.dump(rec, fh, indent=1)
    cl.close()
    sk.close()
    cs.close()
    ctx.close()


if __name__ == "__main__":
    main()
