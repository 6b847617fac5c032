"""lb200_clusters_fill at every launch shape and at its tile, pair-capacity, plane and AtlasSorter edges, bit for bit against the
restatement (oracle/oracle_clusters.c) and, where it is built, the reference's own code (oracle/_ref/libclusters_shim_b200.so), as
tests/test_clusters_gpu.py's check_fill compares them: lights[], clusters[], map[], the AtlasSorter list and the uncast list.

clusters_items_kernel gives block b the items [b * chunk, (b + 1) * chunk), chunk = ceil(n_items / grid), and walks them in tiles of 256:
pass 1 loops over the run, pass 2 scans each tile's pair counts and writes its pairs after the tiles before it.  The default grid is one
block per 256 items the cull can emit, at most every co-resident block, so a block runs more than one tile only past about 270,000
visible items on an H100.  Clusters.setLaunch forces the grid (1, 2, 3, 5, 7, 31, 132, every co-resident block) so that small scenes
reach several tiles per block, kind boundaries inside later tiles and on block boundaries, and blocks without items; lastLaunch reports
the grid and the tiles per block, from which each test proves the case it is named for ran.  The scenes are LOCAL_LIGHT entities only,
placed inside the view so that the cull keeps all of them, with the camera at the origin; the light order is the cull's, read back
through light_entities, and per-light properties are set through it."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import clusters as lc
from lumixengine_b200._lib import LumixB200Error
from oracle import pyclusters as pc
from test_clusters_gpu import check_fill, light_records, points_of, probes

pytestmark = pytest.mark.gpu

TILE = 256
# A NaN fov reaches the priority unchanged on x86, as the device's canonical NaN (bits 0x7fffffff) on the GPU: the same NaN only when it
# has those bits (DESIGN 4.8).  The NaN casters here use them, so that the lists compare byte for byte.
NAN = np.uint32(0x7FFFFFFF).view(np.float32)
HALF_FOV = 1.0472 / 2  # frustum_from_viewport's fov is vertical


class Lights:
    """n LOCAL_LIGHT entities (ids 0 .. n-1) at fp64 positions `pos`, culled with radius `cull_r`; point lights of range `r`; the
    attributes check_fill reads (cl, cam, tr, pl, atlas)."""

    def __init__(self, ctx, pos, r, cull_r=None, seed=0, cast_fraction=0.3):
        rng = np.random.default_rng(seed)
        n = len(pos)
        self.ctx, self.rng, self.n = ctx, rng, n
        self.cam = np.zeros(3)
        self.ids = np.arange(n, dtype=np.int32)
        self.tr = np.zeros(n, lb.TRANSFORM_DTYPE)
        self.tr["pos"] = pos
        q = rng.normal(size=(n, 4))
        self.tr["rot"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
        self.tr["scale"] = 1.0
        self.pl = light_records(rng, n, np.asarray(r, np.float32), cast_fraction)
        self.atlas = np.full(n, -1, np.int32)
        self.cs = lb.CullingSystem(ctx)
        self.cs.add(self.ids, 2, pos, self.pl["range"] if cull_r is None else cull_r)
        self.sk = lb.SortKeys(ctx, n, 1)
        self.sk.setTransforms(self.tr)
        self.cl = lb.Clusters(ctx, n)
        self.cl.setPointLights(self.ids, self.pl)

    def cull(self, w, h, far=2000.0):
        f = view_frustum(w, h, far)
        self.cs.cull_device(f)
        return f

    def fill(self, f, w, h, env=None, refl=None):
        res = self.cl.fillClusters(self.sk, self.cs, lc.make_view(self.cam, f, w, h), env, refl)
        assert res.n_lights == self.n, "the cull left out lights the scene placed inside the view"
        return res

    def order(self, res):
        """Entity of light i of the last fill."""
        return self.cl.read(res)["light_entities"]

    def set_lights(self):
        self.cl.setPointLights(self.ids, self.pl)

    def set_atlas(self, atlas):
        """Atlas entries of every entity to `atlas` (-1 = none), the old ones removed first."""
        old = np.flatnonzero(self.atlas >= 0).astype(np.int32)
        if len(old):
            self.cl.setAtlas(old, np.full(len(old), -1, np.int32))
        self.atlas = np.asarray(atlas, np.int32).copy()
        new = np.flatnonzero(self.atlas >= 0).astype(np.int32)
        if len(new):
            self.cl.setAtlas(new, self.atlas[new])

    def close(self):
        self.cl.close()
        self.sk.close()
        self.cs.close()


def view_frustum(w, h, far=2000.0):
    """A w x h view from the origin down -z."""
    return lb.frustum_from_viewport((0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0472, w, h, 0.1, far)


def in_view(rng, n, w, h, depth=(5.0, 300.0), margin=0.9, log_depth=False):
    """n camera-relative positions well inside a w x h view looking down -z, at depths uniform in `depth` (or in its log)."""
    d = np.exp(rng.uniform(*np.log(depth), n)) if log_depth else rng.uniform(*depth, n)
    t = np.tan(HALF_FOV)
    return np.stack([rng.uniform(-margin, margin, n) * d * t * w / h, rng.uniform(-margin, margin, n) * d * t, -d], 1)


def probes_in_view(rng, n_env, n_refl, w, h):
    env, refl = probes(rng, n_env, n_refl, None)
    env["pos"] = in_view(rng, n_env, w, h, (10.0, 200.0)).astype(np.float32)
    refl["pos"] = in_view(rng, n_refl, w, h, (10.0, 200.0)).astype(np.float32)
    env["outer_range"] = rng.uniform(0.5, 3.0, (n_env, 3)).astype(np.float32)
    refl["half_extents"] = rng.uniform(0.5, 3.0, (n_refl, 3)).astype(np.float32)
    return env, refl


def same_bytes(a, b):
    return all(np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)) for k in ("lights", "clusters", "map", "light_entities"))


def co_resident(ctx):
    """clusters_items_kernel's co-resident blocks, as setLaunch(-1) launches them."""
    S = Lights(ctx, in_view(np.random.default_rng(90), 16, 64, 64), 1.0)
    try:
        S.cl.setLaunch(-1)
        S.fill(S.cull(64, 64), 64, 64)
        return S.cl.lastLaunch()[0]
    finally:
        S.close()


def shape_facts(n_lights, n_env, n_refl, grid):
    """What a grid makes of n items: the cases test_grid_sweep has to reach."""
    n = n_lights + n_env + n_refl
    chunk = -(-n // grid)
    facts = set()
    if -(-chunk // TILE) >= 3:
        facts.add("three tiles in a block")
    runs = [min(chunk, max(0, n - b * chunk)) for b in range(grid)]
    if any(r % TILE for r in runs if r):
        facts.add("a partly full last tile")
    if 0 in runs:
        facts.add("blocks without items")
    for B in (n_lights, n_lights + n_env):  # first env probe, first refl probe
        if 0 < B < n:
            off = B % chunk
            if off >= TILE and off % TILE:
                facts.add("a kind boundary inside a later tile")
            if off == 0:
                facts.add("a kind boundary on a block boundary")
    return facts


# 2303 / 2304 / 2305 lights: at one block the first env probe is item 255, 256 and 257 of tile 8 (counting from its first item);
# 17 env and 13 refl probes put a kind boundary on a block boundary at 132 blocks (chunk 18) for 2304 and 2305 lights.
@pytest.mark.parametrize("n_lights", [2303, 2304, 2305])
def test_grid_sweep(ctx, n_lights):
    """Every grid gives the bytes of the default and of the oracle.  Two views of one cull alternate, so that a fill never finds in
    its scratch what a fill of the same view left there."""
    rng = np.random.default_rng(n_lights)
    views = ((1920, 1080), (1280, 720))
    S = Lights(ctx, in_view(rng, n_lights, 1920, 1080), rng.uniform(0.5, 6.0, n_lights), seed=n_lights)
    try:
        atlas = np.full(n_lights, -1, np.int32)
        atlas[rng.choice(n_lights, 40, replace=False)] = rng.integers(0, 64, 40)
        S.set_atlas(atlas)
        env, refl = probes_in_view(rng, 17, 13, 1920, 1080)
        f = S.cull(1920, 1080)
        limit = co_resident(ctx)
        first, seen = {}, set()
        for blocks in (0, 1, 2, 3, 5, 7, 31, 132, -1, 0):
            S.cl.setLaunch(blocks)
            for w, h in views:
                res = S.fill(f, w, h, env, refl)
                got = check_fill(S, f, res, env, refl, w=w, h=h)
                got["result"] = np.frombuffer(bytes(res), np.uint8)
                grid, tiles = S.cl.lastLaunch()
                want = {0: None, -1: limit}.get(blocks, min(blocks, limit))
                assert want is None or grid == want, f"{blocks} blocks asked, {grid} launched"
                assert tiles == -(-(-(-(n_lights + 17 + 13) // grid)) // TILE)
                seen |= shape_facts(n_lights, 17, 13, grid)
                if (w, h) not in first:
                    first[(w, h)] = got
                assert same_bytes(got, first[(w, h)]) and np.array_equal(got["result"], first[(w, h)]["result"]), f"grid {grid}: not the default's bytes"
        S.cl.setLaunch(0)
        # every light and probe lies inside the view, so each boundary has items with pairs on both sides
        need = {"three tiles in a block", "a partly full last tile", "blocks without items", "a kind boundary inside a later tile"}
        if n_lights != 2303:
            need.add("a kind boundary on a block boundary")
        assert need <= seen, f"not reached: {need - seen}"
    finally:
        S.close()


def test_default_grid_past_one_tile_per_block(ctx):
    """At the default rule a block runs more than one tile once the items outnumber 256 per co-resident block."""
    limit = co_resident(ctx)
    n = 2 * limit * TILE + 77
    rng = np.random.default_rng(91)
    S = Lights(ctx, in_view(rng, n, 1920, 1080, depth=(5.0, 1500.0)), rng.uniform(0.05, 0.4, n), seed=91, cast_fraction=0.2)
    try:
        S.set_atlas(np.where(np.arange(n) < 40, np.arange(n) % 64, -1))
        env, refl = probes_in_view(rng, 5, 4, 1920, 1080)
        f = S.cull(1920, 1080)
        res = S.fill(f, 1920, 1080, env, refl)
        grid, tiles = S.cl.lastLaunch()
        assert grid == limit and tiles >= 2, (grid, tiles)
        check_fill(S, f, res, env, refl, w=1920, h=1080)
    finally:
        S.close()


def far_lights(ctx, n, seed):
    """n lights at one point past the last z plane (10,000) of a 4096 x 4096 view, culled with radius 1: at range 1 none has a pair,
    at range 1e6 one covers all 65,536 clusters."""
    S = Lights(ctx, np.tile([0.0, 0.0, -12000.0], (n, 1)), np.ones(n), cull_r=1.0, seed=seed)
    f = S.cull(4096, 4096, far=20000.0)
    order = S.order(S.fill(f, 4096, 4096))
    return S, f, order


def cover(S, order, positions):
    """Lights at `positions` of the light order over every cluster, the others with range 1."""
    S.pl["range"] = 1.0
    S.pl["range"][order[list(positions)]] = 1e6
    S.set_lights()


@pytest.mark.parametrize("at", [0, 128, 255])
def test_one_item_with_a_tiles_worth_of_pairs(ctx, at):
    """One light with 65,536 pairs among 767 without: in pass 2 every other item of its tile shares its offset or the tile's end."""
    S, f, order = far_lights(ctx, 768, 92)
    try:
        cover(S, order, [TILE + at])
        for blocks in (1, 0):
            S.cl.setLaunch(blocks)
            res = S.fill(f, 4096, 4096)
            assert res.n_map == 65536
            grid, tiles = S.cl.lastLaunch()
            assert (grid, tiles) == ((1, 3) if blocks == 1 else (3, 1))  # the light in tile 1 of one block, or tile 0 of block 1
            got = check_fill(S, f, res, w=4096, h=4096)
            assert (got["clusters"]["lights_count"] == 1).all()
    finally:
        S.close()


def probe_with_pairs(S, f, pairs):
    """An env probe whose sphere the restatement puts into exactly `pairs` clusters of the 4096 x 4096 view."""
    pts = points_of(f)
    for z in np.linspace(-3.0, -40.0, 60):
        env = np.zeros(1, lc.CLUSTER_ENV_PROBE_DTYPE)
        env["pos"] = (0.37 * -z * 0.3, 0.21 * -z * 0.3, z)
        env["outer_range"] = (1e-3, 0.0, 0.0)
        out = pc.fill(pts, 4096, 4096, S.cam, np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 4), np.float32),
                      np.zeros(0, pc.POINT_LIGHT), np.zeros(0, np.int32), env, None)
        if len(out["map"]) == pairs:
            return env
    raise AssertionError(f"no probe position gives {pairs} pairs")


def test_map_room(ctx):
    """The map starts with room for 65,536 pairs: 65,536 fit without growth, 65,537 grow it (eight launches, then four)."""
    S, f, order = far_lights(ctx, 300, 93)
    try:
        cover(S, order, [100])
        pts = points_of(f)
        args = (pts, 4096, 4096, S.cam, order, S.tr["pos"][order], S.tr["rot"][order], S.pl[order], S.atlas[order])
        assert len(pc.fill(*args)["map"]) == 65536
        n0 = ctx.launches
        res = S.fill(f, 4096, 4096)
        assert ctx.launches - n0 == 4 and res.n_map == 65536
        check_fill(S, f, res, w=4096, h=4096)
        env = probe_with_pairs(S, f, 1)
        assert len(pc.fill(*args, env, None)["map"]) == 65537
        for launches in (8, 4):
            n0 = ctx.launches
            res = S.fill(f, 4096, 4096, env)
            assert ctx.launches - n0 == launches and res.n_map == 65537
            check_fill(S, f, res, env, w=4096, h=4096)
    finally:
        S.close()


def test_map_room_overflow_from_block_zero(ctx):
    """On a fresh map, at three blocks of 256 lights, block 0 alone holds 131,072 pairs: the first pair past the room (65,536) is its
    own, and blocks 1 and 2 write only past it.  The fill grows the map, runs again and equals the oracle."""
    S, f, order = far_lights(ctx, 768, 94)
    try:
        cover(S, order, [0, 1, 600])
        S.cl.setLaunch(3)
        for launches in (8, 4):
            n0 = ctx.launches
            res = S.fill(f, 4096, 4096)
            assert S.cl.lastLaunch() == (3, 1)
            assert ctx.launches - n0 == launches and res.n_map == 3 * 65536
            got = check_fill(S, f, res, w=4096, h=4096)
            assert (got["clusters"]["lights_count"] == 3).all()
    finally:
        S.close()


def edge_priorities(rng, k):
    """k priorities: negative, -inf and +inf, subnormal, -0 among +0, ordinary ones, and once k allows it 100 values one ulp apart
    above them all but +inf, so that the 64th and 65th best differ only in their last mantissa bits."""
    p = rng.uniform(-2.0, 0.5, k).astype(np.float32)
    special = np.array([-np.inf, np.inf, 1e-40, -1e-40, 1e-45, 0.0, -0.0, 0.0, -0.0, -3.5, -0.0, 0.0], np.float32)
    idx = rng.permutation(k)
    m = min(k, len(special))
    p[idx[:m]] = special[:m]
    if k >= 200:
        p[idx[m:m + 100]] = np.float32(1.0) + np.arange(100, dtype=np.float32) * np.finfo(np.float32).eps
        assert len(np.unique(p[idx[m:m + 100]])) == 100
    return p


def nearby_lights(ctx, n, seed):
    """n lights at (0, 0, -1) with range 1: distance 1 from the camera, so a caster's priority is exactly its fov (range -1: -fov)."""
    S = Lights(ctx, np.tile([0.0, 0.0, -1.0], (n, 1)), np.ones(n), cull_r=1.0, seed=seed)
    f = S.cull(64, 64)
    order = S.order(S.fill(f, 64, 64))
    return S, f, order


def set_casters(S, order, casters, prio, negate=None):
    """Light order positions `casters` cast with priorities `prio` (a quarter through range -1 where `negate`), the others do not."""
    ents = order[casters]
    flags = S.pl["flags"] & ~np.uint32(lc.CAST_SHADOWS)
    flags[ents] |= lc.CAST_SHADOWS
    S.pl["flags"] = flags
    fov = np.asarray(prio, np.float32).copy()
    r = np.ones(len(ents), np.float32)
    if negate is not None:
        r[negate] = -1.0
        fov[negate] = -fov[negate]
    S.pl["fov"][ents] = fov
    S.pl["range"][:] = 1.0
    S.pl["range"][ents] = r
    S.set_lights()


def fill_checked(S, f):
    res = S.fill(f, 64, 64)
    check_fill(S, f, res, w=64, h=64)
    return res


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1023, 1024, 1025, 2049])
def test_atlas_every_light_a_caster(ctx, n):
    """Light and caster counts at the warp and 1,024-light chunk edges, every light a caster, edge priorities (select path)."""
    S, f, order = nearby_lights(ctx, n, 95 + n)
    try:
        prio = edge_priorities(S.rng, n)
        set_casters(S, order, np.arange(n), prio)
        res = fill_checked(S, f)
        assert res.n_shadow == min(n, 64)
        if n == 64:  # exactly 64 casters, one NaN: the replay keeps all 64
            prio[17] = NAN
            set_casters(S, order, np.arange(n), prio)
            res = fill_checked(S, f)
            assert res.n_shadow == 64 and np.isnan(lc.shadow_list(res)["priority"]).sum() == 1
    finally:
        S.close()


def test_atlas_caster_counts_nan_and_uncast_chunks(ctx):
    """3,100 lights (four chunks of the atlas kernel, the last of 28): caster counts at the warp and chunk edges with edge
    priorities, some negative through a range of -1; uncast lights with an atlas entry only in the last chunk or across a chunk boundary;
    NaN priorities only in the last chunk, as the first caster, and at every caster (replay path).  One fill of each path also at one
    block."""
    n = 3100
    S, f, order = nearby_lights(ctx, n, 96)
    rng = S.rng
    try:
        for j, k in enumerate((1, 63, 64, 65, 1023, 1024, 1025, 2049)):
            uncast = np.arange(3080, 3100) if j % 2 == 0 else np.arange(2030, 2060)  # light order positions
            atlas = np.full(n, -1, np.int32)
            atlas[order[uncast]] = rng.integers(0, 64, len(uncast))
            casters = np.sort(rng.choice(np.setdiff1d(np.arange(n), uncast), k, replace=False))
            S.set_atlas(atlas)
            prio = edge_priorities(rng, k)
            set_casters(S, order, casters, prio, negate=rng.random(k) < 0.25)
            res = fill_checked(S, f)
            assert res.n_shadow == min(k, 64) and res.n_uncast == len(uncast)
            if k == 2049:
                S.cl.setLaunch(1)
                assert same_bytes(S.cl.read(fill_checked(S, f)), S.cl.read(res)) and S.cl.lastLaunch() == (1, 13)
                S.cl.setLaunch(0)
        casters = np.sort(rng.choice(n, 2049, replace=False))
        prio = edge_priorities(rng, 2049)
        last = np.flatnonzero(casters >= 3072)
        for name, nan_at in (("last chunk", [last[len(last) // 2]]), ("first caster", [0]), ("every caster", np.arange(2049))):
            p = prio.copy()
            p[nan_at] = NAN
            set_casters(S, order, casters, p)
            res = fill_checked(S, f)
            assert res.n_shadow == 64, name
            if name == "last chunk":
                S.cl.setLaunch(1)
                assert same_bytes(S.cl.read(fill_checked(S, f)), S.cl.read(res)) and S.cl.lastLaunch()[0] == 1
                S.cl.setLaunch(0)
    finally:
        S.close()


@pytest.mark.parametrize("w,h", [(64, 64), (1920, 1080), (4096, 4096)])
def test_plane_exact_spheres(ctx, w, h):
    """Spheres at exactly dist == r and dist == -r of an x, y or z cluster plane (the restatement's planes for the view, fp32 light
    positions, the camera at the origin so that Vec3(pos - cam) is exact): the device's planes and range() put them where the reference
    does."""
    rng = np.random.default_rng(w + h)
    n = 600
    pos = in_view(rng, n, w, h, depth=(0.3, 400.0), log_depth=True).astype(np.float32)  # every z plane has lights near it
    f = view_frustum(w, h)
    xp, yp, zp = pc.cluster_planes(points_of(f), w, h)
    planes = (xp[:(w + 63) // 64 + 1], yp[:(h + 63) // 64 + 1], zp)
    r = np.zeros(n, np.float32)
    sign = np.zeros((3, n), np.int8)
    for i in range(n):
        a = i % 3
        P, p = planes[a], pos[i]
        d = P[:, 0] * p[0] + P[:, 1] * p[1] + P[:, 2] * p[2] + P[:, 3]  # float32, in planeDist's order
        j = np.argsort(np.abs(d))[rng.integers(0, min(3, len(d)))]  # one of the nearest planes: a small sphere
        r[i] = abs(d[j])
        sign[a, i] = np.sign(d[j])
    for a in range(3):
        assert (sign[a] > 0).any() and (sign[a] < 0).any(), f"axis {a}: no sphere at dist == r or at dist == -r"
    S = Lights(ctx, pos.astype(np.float64), r, seed=w)
    try:
        S.cull(w, h)
        for blocks in (0, 1):
            S.cl.setLaunch(blocks)
            res = S.fill(f, w, h)
            check_fill(S, f, res, w=w, h=h)
    finally:
        S.close()


def test_set_launch_refusals(ctx):
    """setLaunch refuses blocks below -1 and leaves the shape it had; lastLaunch is (0, 0) before the first fill."""
    S = Lights(ctx, in_view(np.random.default_rng(97), 1000, 1920, 1080), 2.0, seed=97)
    try:
        assert S.cl.lastLaunch() == (0, 0)
        f = S.cull(1920, 1080)
        S.fill(f, 1920, 1080)
        default = S.cl.lastLaunch()
        assert default == (4, 1)  # 1,000 items: one block per 256
        S.cl.setLaunch(2)
        for blocks in (-2, -(1 << 31)):
            with pytest.raises(LumixB200Error) as e:
                S.cl.setLaunch(blocks)
            assert e.value.code == lb._lib.ERR_INVALID
        res = S.fill(f, 1920, 1080)
        assert S.cl.lastLaunch() == (2, 2)
        check_fill(S, f, res)
        S.cl.setLaunch(0)
        S.fill(f, 1920, 1080)
        assert S.cl.lastLaunch() == default
    finally:
        S.close()
