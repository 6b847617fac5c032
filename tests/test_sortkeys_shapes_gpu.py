"""createSortKeys on the device (create_keys_kernel, csrc/sortkeys.cu) at every launch shape and at its LOD, pose, group-table and
capacity edges, bit for bit against the oracle (oracle_sortkeys.c) on the same visible ids.

The kernel is one cooperative launch of `grid` blocks of 256 threads that walk the visible list [MESH | DECAL | CURVE_DECAL] grid-stride
in two passes (count, then write at the claimed slots).  SortKeys.setLaunch picks the grid (1, 2, 3, one or two blocks per SM, every
co-resident block) and the L2 prefetch distance; the visible counts put the last renderable before, on and after block and grid-stride
edges, and the largest makes every thread handle several renderables.  Scenes are added to a culling system and culled by an
orthographic view that sees all of them, so the visible ids, and their count per type, are exactly the ones added.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys

pytestmark = pytest.mark.gpu

MESH, DECAL, LIGHT, CURVE = 0, 1, 2, 3
FLT_MAX = np.finfo(np.float32).max
NEVER = 0xffffffff  # Pose::frame before the first claim


def _canon_pairs(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare(got, exp, lod_exp, pf_exp, n_entities):
    """test_sortkeys_gpu._compare: keys / values as a multiset, groups, instance data by renderable, pose / dirty lists, lod and
    Pose::frame state, bit for bit."""
    assert np.all(got["keys"][1:] >= got["keys"][:-1]), "device keys are not sorted"
    gk, gv = _canon_pairs(got["keys"], got["values"])
    ek, ev = _canon_pairs(exp["keys"], exp["values"])
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev), "sort keys / values differ"
    assert np.array_equal(got["group_count"], exp["group_count"]), "group counts differ"
    assert np.array_equal(got["group_offset"], exp["group_offset"]), "group offsets differ"
    go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
    assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo]), "group renderables differ"
    g_of = np.repeat(np.arange(len(exp["group_count"])), exp["group_count"])
    assert np.array_equal(g_of[go], g_of[eo]), "a renderable sits in another group"
    assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo]), "instance data differs"
    assert np.array_equal(np.sort(got["pose_list"]), np.sort(exp["pose_list"])), "pose lists differ"
    assert np.array_equal(np.sort(got["dirty_list"]), np.sort(exp["dirty_list"])), "dirty lists differ"
    assert np.array_equal(got["lod"][:n_entities].view(np.uint32), lod_exp.view(np.uint32)), "lod state differs"
    assert np.array_equal(got["pose_frame"][:n_entities], pf_exp), "Pose::frame state differs"


def _all_visible(ctx, ids, types, pos):
    """A culling system holding exactly these entities, culled by a view that sees them all."""
    cs = lb.CullingSystem(ctx)
    ids = np.asarray(ids, np.int32)
    if len(ids):
        cs.add(ids, np.asarray(types, np.uint8), np.ascontiguousarray(pos[ids]), 0.5)
    _, res = cs.cull_device(lb.frustum_ortho((0.0, 0.0, 2000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 2000.0, 2000.0, 0.0, 4000.0))
    assert res.total == len(ids), f"{res.total} of {len(ids)} entities visible"
    return cs


def _positions(n, seed):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray((rng.random((n, 3)) * 2.0 - 1.0) * np.array([400.0, 100.0, 400.0]))


class Mirror:
    """A SortKeys object and the oracle's copy of the per-entity state it keeps (ModelInstance::lod, Pose::frame).  Every createSortKeys on
    the device is run by the oracle on the same visible ids and the same state, so the state carries over from call to call on both sides."""

    def __init__(self, ctx, sk, max_groups=None, max_keys=None, max_instances=None):
        self.sk = sk
        self.n = len(sk["model_of"])
        self.S = lb.SortKeys(ctx, self.n, max_groups or sk["max_sort_key"] + 1, max_keys=max_keys or 8 * self.n + 64, max_instances=max_instances or 8 * self.n + 64)
        self.S.setModels(sk["models"], sk["meshes"])
        self.lod, self.pf = sk["lod"].copy(), sk["pose_frame"].copy()
        self.upload()
        self.S.setTransforms(sk["transforms"])

    def upload(self):
        """The host state (and the flags, which tests edit) into the device records."""
        sk = self.sk
        self.S.setInstances(sk["model_of"], self.lod, sk["flags"], self.pf, sk["decal_sort_key"], sk["decal_layer"])

    def view(self, frame, is_shadow=False, td=1.0 / 30.0, mult=1.0, max_sort_key=None, camera=(3.0, -2.0, 5.0), ref=(0.0, 0.0, 0.0)):
        sk = self.sk
        return sortkeys.make_view(camera, ref, td, mult, frame, is_shadow, sk["max_sort_key"] if max_sort_key is None else max_sort_key, sk["layer_to_bucket"],
                                  sk["depth_sorted_buckets"])

    def oracle(self, oracle, ids, types, view):
        sk = self.sk
        return oracle.create_sort_keys(ids, types, sk["transforms"], sk["model_of"], self.lod, sk["flags"], self.pf, sk["decal_sort_key"], sk["decal_layer"],
                                       sk["models"], sk["meshes"], view)

    def run(self, oracle, cs, ids, types, view, grid=None, what=""):
        res = self.S.createSortKeys(cs, view)
        got = self.S.read(res)
        exp = self.oracle(oracle, ids, types, view)
        counts = (res.n_keys, res.n_instances, res.n_pose, res.n_dirty)
        assert counts == (len(exp["keys"]), len(exp["group_renderables"]), len(exp["pose_list"]), len(exp["dirty_list"])), what
        try:
            _compare(got, exp, self.lod, self.pf, self.n)
        except AssertionError as e:
            raise AssertionError(f"{what}: {e}") from None
        if grid is not None:
            assert self.S.lastLaunch()[0] == grid, f"{what}: launched {self.S.lastLaunch()[0]} blocks, asked for {grid}"
        return res, exp

    def close(self):
        self.S.close()


# ------------------------------------------------------------------ launch shapes ------------------------------------------------------------------
@pytest.fixture(scope="module")
def big(ctx, oracle):
    """One entity table big enough for four grid strides of every co-resident block, culled in prefixes: `prefix(n)` is a culling system
    whose visible list holds the first n renderables of the table (LOCAL_LIGHTs in between, and three in front of the first renderable).
    -> dict(m=Mirror, limit / limit_hbm = co-resident blocks with the group counters in shared memory / HBM, sms, prefix, types)"""
    # co-resident blocks of either group-table path, from a small scene
    types0 = np.zeros(64, np.uint8)
    pos0 = _positions(64, 1)
    sk0 = scenes.sortkey_setup(64, types0, pos0, seed=3)
    m0 = Mirror(ctx, sk0, max_groups=9000)
    cs0 = _all_visible(ctx, np.arange(64), types0, pos0)
    m0.S.setLaunch(-1)
    m0.S.createSortKeys(cs0, m0.view(1))
    limit, in_smem, _ = m0.S.lastLaunch()
    assert in_smem
    m0.S.createSortKeys(cs0, m0.view(2, max_sort_key=8999))
    limit_hbm, in_smem, _ = m0.S.lastLaunch()
    assert not in_smem
    cs0.close()
    m0.close()
    # the table: ~6 % lights, the rest MESH / DECAL / CURVE_DECAL
    n_ren = 4 * limit * 256 + 77
    n = int(n_ren * 1.07) + 16
    rng = np.random.default_rng(5)
    types = rng.choice(np.array([MESH, DECAL, LIGHT, CURVE], np.uint8), n, p=[0.80, 0.08, 0.06, 0.06]).astype(np.uint8)
    types[:3] = LIGHT
    ren_cum = np.cumsum(types != LIGHT)
    assert ren_cum[-1] >= n_ren
    pos = _positions(n, 6)
    sk = scenes.sortkey_setup(n, types, pos, seed=8)
    m = Mirror(ctx, sk, max_groups=9000)
    cache = {}

    def prefix(k):
        end = 3 if k == 0 else int(np.searchsorted(ren_cum, k)) + 1
        if end not in cache:
            ids = np.arange(end, dtype=np.uint32)
            cache[end] = (_all_visible(ctx, ids, types[:end], pos), ids, types[:end])
        cs, ids, ty = cache[end]
        assert int((ty != LIGHT).sum()) == k
        return cs, ids, ty

    # the default launch on more work than two blocks per SM can take in one stride: 2 blocks per SM
    cs, ids, ty = prefix(n_ren)
    m.S.setLaunch(0, -1)
    m.S.createSortKeys(cs, m.view(3))
    m.oracle(oracle, ids, ty, m.view(3))  # the lod and pose state moved on the device: the tests compare against it
    default_grid, _, prefetch = m.S.lastLaunch()
    assert default_grid % 2 == 0 and default_grid <= limit and prefetch == 0
    out = dict(m=m, limit=limit, limit_hbm=limit_hbm, sms=default_grid // 2, prefix=prefix, frame=[10])
    yield out
    for cs, _, _ in cache.values():
        cs.close()
    m.close()


def _grid(big, name):
    return {"1": 1, "2": 2, "3": 3, "sms": big["sms"], "2sms": 2 * big["sms"], "all": big["limit"]}[name]


def _next_frame(big):
    big["frame"][0] += 1
    return big["frame"][0]


@pytest.mark.parametrize("grid_name", ["1", "2", "3", "sms", "2sms", "all"])
def test_every_grid_and_visible_count(ctx, oracle, big, grid_name):
    m = big["m"]
    m.upload()
    grid = _grid(big, grid_name)
    m.S.setLaunch(-1 if grid_name == "all" else grid, 0)
    stride = grid * 256
    for k in (0, 1, 255, 256, 257, stride, stride + 1, 4 * stride + 77):
        cs, ids, ty = big["prefix"](k)
        res, _ = m.run(oracle, cs, ids, ty, m.view(_next_frame(big)), grid=grid, what=f"grid {grid}, {k} visible")
        if k == 4 * stride + 77:
            assert k > 4 * stride and res.n_keys > stride  # every thread walks several renderables in both passes
    m.S.setLaunch(0, -1)


@pytest.mark.parametrize("prefetch", [1, 2, 4])
@pytest.mark.parametrize("grid_name", ["1", "2sms"])
def test_prefetch_distances(ctx, oracle, big, grid_name, prefetch):
    """prefetch 1 reuses the next id (ahead == stride), 2 and 4 read the id `prefetch` strides ahead."""
    m = big["m"]
    m.upload()
    grid = _grid(big, grid_name)
    m.S.setLaunch(grid, prefetch)
    for k in ((prefetch + 1) * grid * 256 + 13, 4 * grid * 256 + 77):
        cs, ids, ty = big["prefix"](k)
        m.run(oracle, cs, ids, ty, m.view(_next_frame(big)), grid=grid, what=f"grid {grid}, prefetch {prefetch}, {k} visible")
        assert m.S.lastLaunch()[2] == prefetch
    m.S.setLaunch(0, -1)


SEGMENTS = {  # visible MESH, DECAL, CURVE_DECAL, LOCAL_LIGHT
    "meshes_only": (700, 0, 0, 30),
    "decals_only": (0, 700, 0, 30),
    "curve_decals_only": (0, 0, 700, 30),
    "no_meshes": (0, 300, 400, 30),
    "mid_warp_mid_block": (300, 45, 70, 30),  # MESH | DECAL at 300 (block 1, lane 12 of warp 1), DECAL | CURVE at 345
    "block_aligned": (256, 256, 1, 5),
    "lights_only": (0, 0, 0, 40),
}


@pytest.mark.parametrize("segments", list(SEGMENTS))
def test_segment_edges(ctx, oracle, big, segments):
    """The three segments seen as one index space, LOCAL_LIGHT skipped: empty segments and boundaries inside a warp and a block."""
    m = big["m"]
    m.upload()
    counts = SEGMENTS[segments]
    rng = np.random.default_rng(sum(counts))
    types = np.concatenate([np.full(c, t, np.uint8) for c, t in zip(counts, (MESH, DECAL, CURVE, LIGHT))])
    ids = rng.permutation(m.n)[:len(types)].astype(np.uint32)  # ids scattered over the table, types reassigned
    pos = _positions(m.n, 9)
    cs = _all_visible(ctx, ids, types, pos)
    for grid in (1, 2, 3):
        m.S.setLaunch(grid, 0)
        res, exp = m.run(oracle, cs, ids, types, m.view(_next_frame(big)), grid=grid, what=f"{segments}, grid {grid}")
        light_ids = set(ids[types == LIGHT].tolist())
        assert not light_ids & set((exp["values"] & 0xffffffff).tolist())
    m.S.setLaunch(0, -1)
    cs.close()


# ------------------------------------------------------------------ group table ------------------------------------------------------------------
def _group_scene(n_groups, n):
    """n MESH entities of one-mesh models, model i drawing mesh sort key i (auto-instanced, layers 0 / 1 in buckets 0 / 3): with
    n_groups == 1 every instance is in one group; otherwise model_of = id % n_groups, so groups of one and two instances."""
    models = np.zeros(n_groups, sortkeys.SK_MODEL_DTYPE)
    models["lod_distances"] = FLT_MAX
    models["lod_from"], models["lod_to"] = 0, -1
    models["lod_to"][:, 0] = 0
    models["mesh_base"] = np.arange(n_groups)
    models["mesh_count"] = 1
    meshes = np.zeros(n_groups, sortkeys.SK_MESH_DTYPE)
    meshes["sort_key"] = np.arange(n_groups)
    meshes["material_index"] = np.arange(n_groups) * 7 + 1
    meshes["layer"] = np.arange(n_groups) % 2
    n_all = n + 40
    types = np.zeros(n_all, np.uint8)
    types[n:] = LIGHT
    pos = _positions(n_all, n_groups)
    tr = np.zeros(n_all, lb.TRANSFORM_DTYPE)
    tr["pos"] = pos
    tr["rot"] = scenes.random_unit_quats(np.random.default_rng(1), n_all)
    tr["scale"] = 1.5
    sk = dict(models=models, meshes=meshes, model_of=(np.arange(n_all) % n_groups).astype(np.uint32), lod=np.zeros(n_all, np.float32),
              flags=np.zeros(n_all, np.uint8), pose_frame=np.full(n_all, NEVER, np.uint32), decal_sort_key=np.zeros(n_all, np.uint32),
              decal_layer=np.zeros(n_all, np.uint8), transforms=tr, layer_to_bucket=[0, 3], depth_sorted_buckets=(), max_sort_key=n_groups - 1)
    return sk, types, pos


@pytest.mark.parametrize("grid_name", ["1", "2sms"])
@pytest.mark.parametrize("n_groups", [1, 8192, 8193])
def test_group_table_edges(ctx, oracle, big, n_groups, grid_name):
    """1 group that every block adds to, the largest shared-memory group table (8192) and the first HBM one (8193, second barrier)."""
    grid = _grid(big, grid_name)
    n = 3 * 2 * big["sms"] * 256 + 5 if n_groups == 1 else n_groups + 3000
    sk, types, pos = _group_scene(n_groups, n)
    m = Mirror(ctx, sk)
    ids = np.arange(len(types), dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, pos)
    m.S.setLaunch(grid, 0)
    for frame in (1, 2):
        res, exp = m.run(oracle, cs, ids, types, m.view(frame), grid=grid, what=f"{n_groups} groups, grid {grid}")
        assert m.S.lastLaunch()[1] == (n_groups <= 8192)
        assert res.n_instances == n and res.n_groups == n_groups
        if n_groups > 1:
            assert int((exp["group_count"] == 1).sum()) > 1000
    cs.close()
    m.close()


# ------------------------------------------------------------------ LOD edges ------------------------------------------------------------------
def _lod_models():
    """Three hand-built models, squared LOD distances 100 / 400 / 900 / 1600:
    A: five non-empty LODs (LOD 4 has two meshes), B: LOD 1 empty, C: LOD 4 empty (not drawn beyond 40 units)."""
    models = np.zeros(3, sortkeys.SK_MODEL_DTYPE)
    models["lod_distances"] = [100.0, 400.0, 900.0, 1600.0]
    models["lod_from"], models["lod_to"] = 0, -1
    meshes = []

    def mesh(lod, layer):
        meshes.append((len(meshes), 11 * len(meshes) + 3, float(lod), layer, 0, 0))

    # A: meshes 0..5
    models[0]["mesh_base"] = 0
    for l, (f, t) in enumerate([(0, 0), (1, 1), (2, 2), (3, 3), (4, 5)]):
        models[0]["lod_from"][l], models[0]["lod_to"][l] = f, t
    for l, layer in ((0, 0), (1, 0), (2, 1), (3, 3), (4, 0), (4, 3)):
        mesh(l, layer)
    models[0]["mesh_count"] = 6
    # B: meshes 6..9, LOD 1 empty
    models[1]["mesh_base"] = 6
    for l, (f, t) in enumerate([(0, 0), (1, 0), (1, 1), (2, 2), (3, 3)]):
        models[1]["lod_from"][l], models[1]["lod_to"][l] = f, t
    for l, layer in ((0, 0), (2, 0), (3, 1), (4, 3)):
        mesh(l, layer)
    models[1]["mesh_count"] = 4
    # C: meshes 10..13, LOD 4 empty
    models[2]["mesh_base"] = 10
    for l, (f, t) in enumerate([(0, 0), (1, 1), (2, 2), (3, 3), (0, -1)]):
        models[2]["lod_from"][l], models[2]["lod_to"][l] = f, t
    for l, layer in ((0, 0), (1, 3), (2, 0), (3, 0)):
        mesh(l, layer)
    models[2]["mesh_count"] = 4
    return models, np.array(meshes, sortkeys.SK_MESH_DTYPE)


def _lod_scene():
    """Every model at squared distances below, on and above each threshold (also through lod_multiplier 2: x^2 + y^2 = 2 * threshold),
    each with stored lods: the LOD itself, +-0.25 from it, 3.5 and 3.25 (truncate to 3), 2.9, 1.25, 0.5, 4 and 0."""
    models, meshes = _lod_models()
    xy = [(0, 0), (9, 0), (10, 0), (11, 0), (20, 0), (29, 0), (30, 0), (31, 0), (40, 0), (41, 0), (60, 0), (10, 10), (20, 20), (30, 30), (40, 40), (15, 0)]
    stored = ["idx", "+", "-", 3.5, 3.25, 2.9, 1.25, 0.5, 4.0, 0.0]
    rows = []
    for mi in range(3):
        for x, y in xy:
            d2 = float(x * x + y * y)
            idx = float(sum(d2 >= t for t in (100.0, 400.0, 900.0, 1600.0)))
            for s in stored:
                lod = idx if s == "idx" else idx + 0.25 if s == "+" else idx - 0.25 if s == "-" else s
                rows.append((mi, x, y, lod))
    n = len(rows)
    tr = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr["pos"] = [(float(x), float(y), 0.0) for _, x, y, _ in rows]
    tr["rot"] = scenes.random_unit_quats(np.random.default_rng(2), n)
    tr["scale"] = 0.75
    sk = dict(models=models, meshes=meshes, model_of=np.array([r[0] for r in rows], np.uint32), lod=np.array([r[3] for r in rows], np.float32),
              flags=np.zeros(n, np.uint8), pose_frame=np.full(n, NEVER, np.uint32), decal_sort_key=np.zeros(n, np.uint32), decal_layer=np.zeros(n, np.uint8),
              transforms=tr, layer_to_bucket=[0, 1, 0xff, 2], depth_sorted_buckets=(1,), max_sort_key=int(meshes["sort_key"].max()))
    return sk


@pytest.mark.parametrize("grid", [1, 2])
def test_lod_smoothing_edges(ctx, oracle, grid):
    sk = _lod_scene()
    n = len(sk["model_of"])
    types = np.zeros(n, np.uint8)
    ids = np.arange(n, dtype=np.uint32)
    pos = np.ascontiguousarray(sk["transforms"]["pos"])
    cs = _all_visible(ctx, ids, types, pos)
    quarter = np.float32(0.25)
    below = np.nextafter(quarter, np.float32(0))  # |d| = 0.25 is one ulp above the time delta: a step, not a snap
    lod0 = sk["lod"].copy()
    # |d| == time_delta: every +-0.25 entity snaps to its LOD
    m = Mirror(ctx, sk)
    m.S.setLaunch(grid, 0)
    m.run(oracle, cs, ids, types, m.view(1, td=quarter), grid=grid, what="time_delta 0.25")
    snapped = np.abs(lod0 - m.lod) == 0.25
    assert snapped.sum() > 50
    # the same start one ulp below: a step, two LODs drawn; then the state carries over through the other edges
    m.lod[:] = lod0
    m.upload()
    frames = [dict(td=below), dict(td=0.0), dict(td=quarter, mult=2.0), dict(td=0.1, is_shadow=True), dict(td=1.0 / 30.0, mult=1.25),
              dict(td=0.5), dict(td=quarter, mult=2.0)]
    for f, kw in enumerate(frames):
        before = m.lod.copy()
        m.run(oracle, cs, ids, types, m.view(2 + f, **kw), grid=grid, what=f"frame {f}: {kw}")
        if f == 0:
            assert np.any((np.abs(lod0 - m.lod) > 0.24) & (np.abs(lod0 - m.lod) < 0.25))  # stepped by a hair less than 0.25
        if kw.get("is_shadow"):
            assert np.any((before == m.lod) & (before != np.floor(before)))  # a shadow view snaps, never steps: fractional lods stay
        if kw.get("td") == 0.0:
            assert np.array_equal(before.view(np.uint32), m.lod.view(np.uint32))
    assert np.any((m.lod > 3.0) & (m.lod < 4.0))  # some instance still holds a lod that truncates to 3
    cs.close()
    m.close()


# ------------------------------------------------------------------ pose claim and flags ------------------------------------------------------------------
def _flags_scene(n=900, seed=4):
    """Skinned and plain models whose meshes sit on every kind of layer (layer_to_bucket [0, 1, 0xff, 2], bucket 1 depth-sorted): a skinned
    mesh on a layer the view does not have, depth-sorted skinned / MOVED / decal renderables; flags cycle through none, MOVED, dirty and
    MOVED + dirty; some instances already claimed this frame."""
    models = np.zeros(3, sortkeys.SK_MODEL_DTYPE)
    models["lod_distances"] = FLT_MAX
    models["lod_from"], models["lod_to"] = 0, -1
    models["lod_to"][:, 0] = [2, 3, 0]
    models["mesh_base"] = [0, 3, 7]
    models["mesh_count"] = [3, 4, 1]
    meshes = np.zeros(8, sortkeys.SK_MESH_DTYPE)
    meshes["sort_key"] = np.arange(8) * 5 + 2
    meshes["material_index"] = np.arange(8) + 100
    meshes["layer"] = [0, 1, 2, 0, 1, 2, 3, 0]
    meshes["skinned"] = [1, 1, 1, 0, 0, 0, 0, 1]
    rng = np.random.default_rng(seed)
    types = rng.choice(np.array([MESH, DECAL, LIGHT, CURVE], np.uint8), n, p=[0.8, 0.1, 0.05, 0.05]).astype(np.uint8)
    pos = _positions(n, seed)
    tr = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr["pos"] = pos
    tr["rot"] = scenes.random_unit_quats(rng, n)
    tr["scale"] = rng.uniform(0.5, 2.0, (n, 3)).astype(np.float32)
    flags = np.array([0, sortkeys.MOVED, sortkeys.DIRTY, sortkeys.MOVED | sortkeys.DIRTY, 0, sortkeys.MOVED], np.uint8)[np.arange(n) % 6]
    sk = dict(models=models, meshes=meshes, model_of=(np.arange(n) % 3).astype(np.uint32), lod=np.zeros(n, np.float32), flags=flags,
              pose_frame=np.full(n, NEVER, np.uint32), decal_sort_key=rng.integers(0, 5000, n).astype(np.uint32),
              decal_layer=(np.arange(n) % 4).astype(np.uint8), transforms=tr, layer_to_bucket=[0, 1, 0xff, 2], depth_sorted_buckets=(1,),
              max_sort_key=int(meshes["sort_key"].max()) + 4)
    return sk, types, pos


@pytest.mark.parametrize("grid", [0, 1])
def test_pose_claim_across_views_of_one_frame(ctx, oracle, grid):
    """A main and a shadow view of one frame claim every skinned instance once; the next frame claims again, also across the
    % 0xffffffff wrap of the frame number.  Dirty + skinned instances go to the dirty list and claim nothing."""
    sk, types, pos = _flags_scene()
    F = 0xfffffffe
    sk["pose_frame"][::7] = F  # already claimed in this frame
    m = Mirror(ctx, sk)
    m.S.setLaunch(grid, 0)
    ids = np.arange(len(types), dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, pos)
    skinned = np.isin(sk["model_of"], [0, 2]) & (types == MESH)
    dirty = (sk["flags"] & sortkeys.DIRTY) != 0
    for frame, shadow, claims in ((F, False, True), (F, True, False), (F, False, False), (F + 1, True, True), (F + 1, False, False),
                                  (F + 2, False, True), (7, True, True), (7, True, False)):
        res, exp = m.run(oracle, cs, ids, types, m.view(frame, is_shadow=shadow), what=f"frame {frame:#x}, shadow {shadow}")
        assert (res.n_pose > 0) == claims, f"frame {frame:#x}: {res.n_pose} claims"
        assert not np.isin(exp["pose_list"], np.nonzero(dirty)[0]).any()
        assert res.n_dirty == int((dirty & (types == MESH)).sum())
    assert skinned.sum() > 100
    cs.close()
    m.close()


@pytest.mark.parametrize("is_shadow", [False, True])
@pytest.mark.parametrize("grid", [0, 1, 3])
def test_flags_by_view_kind(ctx, oracle, grid, is_shadow):
    """MOVED draws a plain key in a main view and is auto-instanced in a shadow view; MOVED + skinned stays skinned; a skinned mesh on a
    layer the view does not have keeps its key with bucket 0xff; depth-sorted buckets (0x101) go into the key truncated to 8 bits."""
    sk, types, pos = _flags_scene(seed=6)
    m = Mirror(ctx, sk)
    m.S.setLaunch(grid, 0)
    ids = np.arange(len(types), dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, pos)
    res, exp = m.run(oracle, cs, ids, types, m.view(3, is_shadow=is_shadow), what=f"grid {grid}, shadow {is_shadow}")
    buckets = exp["keys"] >> np.uint64(56)
    assert (buckets == 0xff).any() and (buckets == 1).any()
    cs.close()
    m.close()


# ------------------------------------------------------------------ capacities ------------------------------------------------------------------
def test_capacities_exact_and_one_short(ctx, oracle):
    """max_keys / max_instances equal to what the view emits pass; one less is LB200_ERR_CAPACITY, and the next (smaller) view on the
    same object matches the oracle, which went through both calls."""
    n = 4000
    types = np.random.default_rng(3).choice(np.array([MESH, DECAL, LIGHT, CURVE], np.uint8), n, p=[0.85, 0.07, 0.03, 0.05]).astype(np.uint8)
    pos = _positions(n, 3)
    sk = scenes.sortkey_setup(n, types, pos, seed=12)
    ids = np.arange(n, dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, pos)
    half = ids[: n // 2]
    cs_half = _all_visible(ctx, half, types[: n // 2], pos)
    probe = Mirror(ctx, sk)
    exp = probe.oracle(oracle, ids, types, probe.view(1))
    probe.close()
    nk, ni = len(exp["keys"]), len(exp["group_renderables"])
    assert nk > 1000 and ni > 1000
    for max_keys, max_instances, fits in ((nk, ni, True), (nk - 1, ni, False), (nk, ni - 1, False)):
        m = Mirror(ctx, sk, max_keys=max_keys, max_instances=max_instances)
        what = f"max_keys {max_keys} / max_instances {max_instances} for {nk} / {ni}"
        if fits:
            m.run(oracle, cs, ids, types, m.view(1), what=what)
        else:
            with pytest.raises(lb.LumixB200Error) as err:
                m.S.createSortKeys(cs, m.view(1))
            assert err.value.code == _lib.ERR_CAPACITY, what
            m.oracle(oracle, ids, types, m.view(1))  # the lod and pose state moved on the device too
        res, _ = m.run(oracle, cs_half, half, types[: n // 2], m.view(2), what=f"{what}, the call after")
        assert res.n_keys <= max_keys and res.n_instances <= max_instances
        m.close()
    cs.close()
    cs_half.close()


# ------------------------------------------------------------------ moved instances ------------------------------------------------------------------
def test_move_batches_and_end_frame(ctx, oracle):
    """onModelInstanceMoved / endFrame sequences: two batches before one endFrame (the later transform wins), an id >= max_entities
    (record skipped, sphere written), endFrame twice, a move after endFrame (MOVED again), endFrame before any move."""
    n = 800
    types = np.random.default_rng(8).choice(np.array([MESH, DECAL, LIGHT, CURVE], np.uint8), n, p=[0.85, 0.05, 0.05, 0.05]).astype(np.uint8)
    pos = _positions(n, 8)
    sk = scenes.sortkey_setup(n, types, pos, seed=13, moved_fraction=0.0, dirty_fraction=0.0)
    m = Mirror(ctx, sk)
    ids = np.arange(n, dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, pos)
    rng = np.random.default_rng(21)
    mesh_ids = np.nonzero(types == MESH)[0]
    pick = rng.choice(mesh_ids, 240, replace=False).astype(np.int32)
    A, B, C, D = pick[:60], pick[60:120], pick[120:180], pick[180:]
    zero_prev = m.S.prevTransforms()
    assert not zero_prev["pos"].any()
    fresh = lb.SortKeys(ctx, 16, 4)
    fresh.endFrame()  # before any move: nothing to do
    assert not fresh.prevTransforms()["pos"].any()
    fresh.close()

    def transforms(k, seed):
        r = np.random.default_rng(seed)
        t = np.zeros(k, lb.TRANSFORM_DTYPE)
        t["pos"] = (r.random((k, 3)) * 2.0 - 1.0) * 300.0
        t["rot"] = scenes.random_unit_quats(r, k)
        t["scale"] = r.uniform(0.5, 2.0, (k, 3)).astype(np.float32)
        return t

    def move(ents, tr, seed):
        k = len(ents)
        br = np.random.default_rng(seed).uniform(0.5, 3.0, k).astype(np.float32)
        dev = [ctx.to_device(np.ascontiguousarray(ents, np.int32)), ctx.to_device(tr), ctx.to_device(br), ctx.to_device(np.zeros((k, 3))),
               ctx.to_device(np.zeros(k, np.float32))]
        m.S.moveDevice(dev[0], dev[1], k, dev[2], dev[3], dev[4])
        got_pos, got_rad = ctx.copy_to_host(dev[3], 3 * k, np.float64).reshape(k, 3), ctx.copy_to_host(dev[4], k, np.float32)
        for p in dev:
            ctx.free_device(p)
        assert np.array_equal(got_pos, tr["pos"]), "spheres: positions"
        assert np.array_equal(got_rad.view(np.uint32), (br * tr["scale"].max(axis=1)).astype(np.float32).view(np.uint32)), "spheres: radii"
        valid = ents < n
        sk["transforms"][ents[valid]] = tr[valid]
        sk["flags"][ents[valid]] |= sortkeys.MOVED

    def end_frame():
        m.S.endFrame()
        moved = (sk["flags"] & sortkeys.MOVED) != 0
        expected_prev[moved] = sk["transforms"][moved]
        sk["flags"][moved] &= ~np.uint8(sortkeys.MOVED)
        got = m.S.prevTransforms()
        for field in ("pos", "rot", "scale"):
            assert got[field].tobytes() == expected_prev[field].tobytes(), f"prev_frame_transform: {field}"

    expected_prev = np.zeros(n, lb.TRANSFORM_DTYPE)
    frame = [0]

    def draw(what):
        frame[0] += 1
        for shadow in (False, True):
            m.run(oracle, cs, ids, types, m.view(frame[0], is_shadow=shadow), what=what)

    b1 = np.concatenate([A, B])
    move(b1, transforms(len(b1), 1), 1)
    b2 = np.concatenate([B, C, np.array([n + 5, n], np.int32)])  # ids >= max_entities: sphere only
    move(b2, transforms(len(b2), 2), 2)
    draw("two batches")
    end_frame()
    draw("after endFrame")
    end_frame()  # twice: nothing moved since the last one
    draw("after a second endFrame")
    b3 = np.concatenate([D, A])
    move(b3, transforms(len(b3), 3), 3)
    draw("moved after endFrame")
    end_frame()
    draw("after the last endFrame")
    cs.close()
    m.close()


# ------------------------------------------------------------------ host-side checks ------------------------------------------------------------------
def test_entity_ids_beyond_max_entities_are_rejected(ctx, oracle):
    """A culling system holding an id >= max_entities is refused before anything is launched; the largest id that fits runs."""
    n = 300
    types = np.zeros(n + 1, np.uint8)
    pos = _positions(n + 1, 2)
    sk = scenes.sortkey_setup(n, types[:n], pos[:n], seed=4)
    m = Mirror(ctx, sk)
    ids = np.arange(n, dtype=np.uint32)
    cs = _all_visible(ctx, ids, types[:n], pos)
    m.run(oracle, cs, ids, types[:n], m.view(1), what="ids up to max_entities - 1")
    cs_bad = _all_visible(ctx, np.arange(n + 1, dtype=np.uint32), types, pos)
    launches = ctx.launches
    with pytest.raises(lb.LumixB200Error) as err:
        m.S.createSortKeys(cs_bad, m.view(2))
    assert err.value.code == _lib.ERR_INVALID and ctx.launches == launches
    with pytest.raises(lb.LumixB200Error) as err:  # a view whose max_sort_key is below a mesh's sort key
        m.S.createSortKeys(cs, m.view(2, max_sort_key=sk["max_sort_key"] - 1))
    assert err.value.code == _lib.ERR_INVALID and ctx.launches == launches
    m.run(oracle, cs, ids, types[:n], m.view(3), what="after the refusals")
    cs.close()
    cs_bad.close()
    m.close()


@pytest.mark.parametrize("model,field,lod,value", [
    (0, "lod_to", 4, 6),     # one past the model's 6 meshes
    (1, "lod_from", 3, -1),  # a negative first mesh
])
def test_set_models_rejects_lod_ranges_outside_the_model(ctx, model, field, lod, value):
    models, meshes = _lod_models()
    S = lb.SortKeys(ctx, 8, 256)
    S.setModels(models, meshes)  # every range inside: accepted
    bad = models.copy()
    bad[model][field][lod] = value
    with pytest.raises(lb.LumixB200Error) as err:
        S.setModels(bad, meshes)
    assert err.value.code == _lib.ERR_INVALID
    ok = models.copy()
    ok[1]["lod_from"][1], ok[1]["lod_to"][1] = 7, -3  # empty ranges are never read, wherever they point
    S.setModels(ok, meshes)
    S.close()


@pytest.mark.parametrize("field,value,n_meshes", [
    ("mesh_count", 5, 14),  # model C's meshes [10, 15) leave the 14-mesh table
    ("mesh_base", 11, 14),  # [11, 15)
    (None, None, 12),       # the whole table cut short: C's [10, 14) leaves 12 meshes
])
def test_create_keys_refuses_models_past_the_mesh_table(ctx, oracle, field, value, n_meshes):
    """A model table may be set ahead of the mesh table it will be paired with, but nothing is launched while a model's meshes leave the
    mesh table; once both fit, the same object runs and matches the oracle."""
    sk = _lod_scene()
    m = Mirror(ctx, sk)
    n = len(sk["model_of"])
    types = np.zeros(n, np.uint8)
    ids = np.arange(n, dtype=np.uint32)
    cs = _all_visible(ctx, ids, types, np.ascontiguousarray(sk["transforms"]["pos"]))
    bad = sk["models"].copy()
    if field is not None:
        bad[2][field] = value
    m.S.setModels(bad, sk["meshes"][:n_meshes])
    launches = ctx.launches
    with pytest.raises(lb.LumixB200Error) as err:
        m.S.createSortKeys(cs, m.view(1))
    assert err.value.code == _lib.ERR_INVALID and ctx.launches == launches
    m.S.setModels(sk["models"], sk["meshes"])
    m.run(oracle, cs, ids, types, m.view(2), what="after the tables fit again")
    cs.close()
    m.close()


def test_set_launch_rejects_other_values(ctx):
    S = lb.SortKeys(ctx, 8, 4)
    assert S.lastLaunch() == (0, False, 0)
    for blocks, prefetch in ((-2, -1), (0, 5), (0, -2), (-7, 0)):
        with pytest.raises(lb.LumixB200Error):
            S.setLaunch(blocks, prefetch)
    S.setLaunch(-1, 4)
    S.setLaunch(100000, 0)  # more blocks than are co-resident: the launch takes what fits
    S.close()
