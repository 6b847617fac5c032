"""Several views culled in one pass (CullingSystem.cull_views, csrc/cull_views_kernel.cuh), held to the oracle view by view.

Every view of a call is compared with oracle.OracleCulling.cull of that view alone on the same edits: the visible set per renderable type,
the six statistics, and the visibility rows of the view's mask decoded through the page table after select_view + read_bitmask.  Where the
device holds the page state (device re-binning, device adds / removes) the page layout differs from the oracle's by design: there the
visible sets are held to the oracle and the statistics and mask rows to a lone cull_device of the same view.  The algorithmic bytes of a
call are held to 32 B per page + 16 B per sphere of the pages some view tests + per view 8 B per visible id and 32 B per page.
"""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys

pytestmark = pytest.mark.gpu

STATS = ("pages_tested", "pages_inside", "pages_outside", "pages_filtered", "entities_tested", "entities_inside")
CELL = 300.0
ALL = lb.culling.TYPE_ALL


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Expect:
    """The oracle's answer for one (scene, view, type)."""

    def __init__(self, oc, f, type=ALL):
        self.ids, self.tys, self.st = oc.cull(lb.culling.frustum_bytes(f), -1 if type == ALL else type)
        self.key = np.sort(self.ids.astype(np.int64) * 256 + self.tys)


class ViewResult:
    """One view of a cull_views call (or a cull_device) read back: ids grouped per type, counts and statistics."""

    def __init__(self, ctx, ptr, raw):
        self.raw = raw
        self.total = int(raw.total)
        cnt = np.ctypeslib.as_array(raw.type_count).copy()
        off = np.ctypeslib.as_array(raw.type_offset).copy()
        ts = [int(t) for t in np.nonzero(cnt)[0]]
        self.ids = np.concatenate([ctx.copy_to_host(ptr + 4 * int(off[t]), int(cnt[t]), np.uint32) for t in ts]) if ts else np.zeros(0, np.uint32)
        self._types = np.concatenate([np.full(int(cnt[t]), t, np.uint8) for t in ts]) if ts else np.zeros(0, np.uint8)
        self.stats = {k: int(getattr(raw, k)) for k in STATS}

    def types(self):
        return self._types

    def key(self):
        return np.sort(self.ids.astype(np.int64) * 256 + self._types)


def _check(res, exp, what, stats=True):
    got = np.sort(res.ids.astype(np.int64) * 256 + res.types())
    assert res.total == len(exp.ids) and np.array_equal(got, exp.key), f"{what}: {res.total} visible, oracle {len(exp.ids)}"
    if stats:
        for k in STATS:
            assert res.stats[k] == exp.st[k], f"{what}: {k} {res.stats[k]}, oracle {exp.st[k]}"


class Table:
    """m_cells of a culling system as arrays: entity id per page slot (-1 beyond the count), to decode read_bitmask() rows."""

    def __init__(self, cs):
        pages = cs.pages()
        self.count = np.array([p["count"] for p in pages])
        self.type = np.array([p["type"] for p in pages], np.int64)
        self.ent = np.full((len(pages), 256), -1, np.int64)
        for i, p in enumerate(pages):
            self.ent[i, :p["count"]] = p["entities"]
        self.live = np.arange(256)[None, :] < self.count[:, None]

    def decode(self, mask, what):
        bits = np.unpackbits(mask.view(np.uint8), bitorder="little").reshape(-1, 256).astype(bool)
        assert not (bits & ~self.live).any(), f"{what}: mask bits at or beyond a page's count"
        return np.sort(self.ent[bits] * 256 + np.broadcast_to(self.type[:, None], bits.shape)[bits])


def _frame(cs, ctx, frusta, types=None):
    out = cs.cull_views(frusta, types)
    return [ViewResult(ctx, p, r) for p, r in out], cs.last_algorithmic_bytes()


def _check_call(cs, ctx, oc, frusta, types=None, what="", table=None, stats=True):
    """One cull_views call against the oracle view by view, masks through select_view; -> (results, algorithmic bytes)."""
    types_ = list(types) if types is not None else [ALL] * len(frusta)
    exps = [Expect(oc, f, t) for f, t in zip(frusta, types_)]
    res, nbytes = _frame(cs, ctx, frusta, types)
    table = table or Table(cs)
    for v, (r, e) in enumerate(zip(res, exps)):
        _check(r, e, f"{what} view {v}", stats)
        cs.select_view(v)
        assert np.array_equal(table.decode(cs.read_bitmask(), f"{what} view {v}"), e.key), f"{what} view {v}: mask rows"
    return res, nbytes


def _lone_streamed(cs, f, t=ALL):
    """Spheres a lone cull of the view reads, from its algorithmic bytes."""
    _, r = cs.cull_device(f, t)
    return (cs.last_algorithmic_bytes() - 64 * _pages(cs) - 8 * int(r.total)) // 16


def _pages(cs):
    return int(max(cs.page_ids()) + 1)


def _union_streamed(cs, res, nbytes):
    """Spheres a cull_views call read (each tested page once), from its algorithmic bytes."""
    p = _pages(cs)
    rest = nbytes - 32 * p - sum(8 * r.total + 32 * p for r in res)
    assert rest >= 0 and rest % 16 == 0, rest
    return rest // 16


# ---------------------------------------------------------------- scenes ---------------------------------------------------------------

N_GRID_PAGES = 3584


def _grid_scene(seed=7):
    """1,792 cells (32 in x by 56 in z) with two pages each of different renderable types, 1..40 entities (every fourth cell 1..200);
    the second page of every 17th cell is_big."""
    rng = np.random.default_rng(seed)
    tys, pos, rad = [], [], []
    for c in range(N_GRID_PAGES // 2):
        i, j = c % 32, c // 32
        for k in range(2):
            n = int(rng.integers(1, 201)) if c % 4 == 0 else int(rng.integers(1, 41))
            big = k == 1 and c % 17 == 0
            pos.append(np.stack([(i + 1) * CELL + rng.uniform(5, 295, n), rng.uniform(5, 295, n), (j + 1) * CELL + rng.uniform(5, 295, n)], 1))
            rad.append(rng.uniform(301, 420, n) if big else rng.uniform(0.5, 8.0, n))
            tys.append(np.full(n, (c + k) % 3, np.uint8))
    pos, rad, tys = np.concatenate(pos), np.concatenate(rad).astype(np.float32), np.concatenate(tys)
    return dict(entities=np.arange(len(pos), dtype=np.int32), types=tys, pos=pos, radius=rad)


def _grid_views():
    p = lambda pos, d, far: lb.frustum_perspective(pos, d, (0.0, 1.0, 0.0), 1.2, 1.0, 0.5, far)  # noqa: E731
    return [p((5100.0, 150.0, -200.0), (0.0, 0.0, 1.0), 9000.0),     # across the grid: inside, tested and outside pages
            p((5100.0, 150.0, -200.0), (0.0, 0.0, 1.0), 3000.0),     # nested in the first
            p((4000.0, 150.0, 20000.0), (0.0, 0.0, -1.0), 6000.0),   # from the other end, overlapping the far half
            p((1e6, 0.0, 1e6), (0.0, 0.0, 1.0), 100.0),               # nothing
            lb.frustum_ortho((5000.0, 2000.0, 8000.0), (0.0, -1.0, 0.0), (0.0, 0.0, 1.0), 3000.0, 3000.0, 0.0, 4000.0),
            p((300.0, 150.0, 8000.0), (1.0, 0.0, 0.0), 4000.0),
            p((5100.0, 150.0, -200.0), (0.0, 0.0, 1.0), 9000.0),     # identical to the first
            p((9000.0, 500.0, 8500.0), (-0.6, -0.1, 0.5), 5000.0)]


def _both(ctx, oracle, scene):
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    return cs, oc


@pytest.fixture(scope="module")
def grid(ctx, oracle):
    cs, oc = _both(ctx, oracle, _grid_scene())
    assert cs.page_count() == N_GRID_PAGES
    yield cs, oc, Table(cs)
    cs.close()


@pytest.fixture(scope="module")
def c1(ctx, oracle):
    cs, oc = _both(ctx, oracle, scenes.c1_scene())
    yield cs, oc, Table(cs)
    cs.close()


def _c1_views():
    a = scenes.c1_frustum_args()
    main = lb.frustum_perspective(**a)
    cascades = [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(a, (0.3, -0.8, 0.2), (30.0, 150.0, 600.0, 1500.0))]
    return [main] + cascades + [lb.frustum_perspective(**dict(a, direction=(0.0, 0.0, 1.0))),                              # disjoint
                                lb.frustum_perspective(**dict(a, position=(0.0, 0.0, -300.0), far=400.0)),                  # nested
                                lb.frustum_perspective(**dict(a, position=(1e6, 0.0, 0.0)))]                                # empty


# ---------------------------------------------------------------- view counts and overlap ----------------------------------------------

@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_view_counts_on_c1(ctx, c1, n):
    cs, oc, table = c1
    views = _c1_views()
    res, nbytes = _check_call(cs, ctx, oc, views[:n], what=f"c1 {n} views", table=table)
    lone = [_lone_streamed(cs, f) for f in views[:n]]
    u = _union_streamed(cs, res, nbytes)
    assert max(lone) <= u <= sum(lone), (u, lone)
    ll = cs.lastLaunch()
    assert ll["chunk"] <= min(256, 512 // n) and ll["plane_masking"], ll


@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_view_counts_on_grid(ctx, grid, n):
    cs, oc, table = grid
    views = _grid_views()
    _check_call(cs, ctx, oc, views[:n], what=f"grid {n} views", table=table)
    rev = views[:n][::-1]
    _check_call(cs, ctx, oc, rev, what=f"grid {n} views reversed", table=table)


def test_identical_views_read_rows_once(ctx, c1):
    cs, oc, table = c1
    main = _c1_views()[0]
    for n in (2, 5, 8):
        res, nbytes = _check_call(cs, ctx, oc, [main] * n, what=f"{n} identical", table=table)
        assert _union_streamed(cs, res, nbytes) == _lone_streamed(cs, main) > 0
        assert all(np.array_equal(r.key(), res[0].key()) for r in res)


def test_one_view_runs_the_single_kernel(ctx, grid):
    """n_views = 1: the single cull's kernel and launch rule (chunk up to 256), into view 0's buffers; same bytes as a lone cull."""
    cs, oc, table = grid
    f = _grid_views()[0]
    for blocks, chunk in ((0, 0), (3, 7), (1, 256)):
        cs.setLaunch(blocks, chunk)
        res, nbytes = _check_call(cs, ctx, oc, [f], what=f"one view blocks {blocks} chunk {chunk}", table=table)
        if chunk:
            assert cs.lastLaunch()["chunk"] == chunk
        _, lone = cs.cull_device(f)
        assert nbytes == cs.last_algorithmic_bytes()
    cs.setLaunch()


# ---------------------------------------------------------------- one page, different classes per view ---------------------------------

EDGE_COUNTS = (1, 31, 32, 33, 127, 128, 129, 160, 199, 200, 201, 400)


def _edge_scene():
    """One cell per count in EDGE_COUNTS at x-index 0 (x in [0, 300)), one after another in z; slots alternate 20 m left and right of
    x = 150; two is_big cells at x-index 1."""
    rng = np.random.default_rng(17)
    tys, pos, rad = [], [], []
    for k, n in enumerate(EDGE_COUNTS):
        x = np.where(np.arange(n) % 2 == 0, 130.0, 170.0)
        pos.append(np.stack([x, rng.uniform(10, 290, n), (k + 1) * CELL + rng.uniform(10, 290, n)], 1))
        rad.append(rng.uniform(1.0, 5.0, n))
        tys.append(np.full(n, k % 3, np.uint8))
    for k, n in enumerate((129, 200)):
        vis = np.arange(n) % 2 == 0
        pos.append(np.stack([np.where(vis, 320.0, 590.0), rng.uniform(10, 290, n), (k + 1) * CELL + rng.uniform(10, 290, n)], 1))
        rad.append(np.where(vis, 400.0, 301.0 + rng.uniform(0, 1, n)))
        tys.append(np.full(n, 1 + k, np.uint8))
    pos, rad, tys = np.concatenate(pos), np.concatenate(rad).astype(np.float32), np.concatenate(tys)
    return dict(entities=np.arange(len(pos), dtype=np.int32), types=tys, pos=pos, radius=rad)


def _x_cut(x, inside_below, cz, extent=6000.0):
    """Ortho view whose inside is x <= x (inside_below) or x >= x, `extent` wide in x and z, y in +-5000."""
    px = x - extent / 2 if inside_below else x + extent / 2
    for _ in range(4):
        f = lb.frustum_ortho((px, -5000.0, cz), (0.0, -1.0, 0.0), (0.0, 0.0, 1.0), extent / 2, extent / 2, 0.0, 10000.0)
        i = [p for p in range(6) if (f.xs[p] < -0.99 if inside_below else f.xs[p] > 0.99)]
        edge = f.origin[0] + f.ds[i[0]] if inside_below else f.origin[0] - f.ds[i[0]]
        if abs(edge - x) < 1e-3:
            return f
        px += x - edge
    raise AssertionError(f"ortho view edge at {edge}, wanted {x}")


def _edge_views():
    cz = (len(EDGE_COUNTS) + 2) * CELL / 2
    return {"copy": _x_cut(1000.0, True, cz),    # holds the shifted box of x-index 0: COPY
            "test": _x_cut(150.0, True, cz),     # cuts every cell: TEST
            "skip": _x_cut(5000.0, False, cz),   # beyond every cell but the is_big ones: SKIP
            "masked": _x_cut(450.0, True, cz),   # holds the cells, not their shifted boxes: TEST with an empty plane mask
            "edge": _x_cut(300.01, False, cz)}   # inside the cheap pass's margin of x-index 0: skipped by the exact pass only


def test_same_page_different_classes(ctx, oracle):
    cs, oc = _both(ctx, oracle, _edge_scene())
    table = Table(cs)
    v = _edge_views()
    # the second call follows one whose view 1 worked the x-index 0 pages: view 1's rows of them have to be zeroed again
    calls = {"copy/test/skip/masked": ["copy", "test", "skip", "masked"],
             "zero rows after work": ["test", "edge", "copy"],
             "only the masked view takes them": ["masked", "skip"],
             "test twice": ["test", "skip", "test", "masked", "test"]}
    for shape in ((0, 0), (1, 7), (3, 1), (2, 33)):
        cs.setLaunch(*shape)
        for name, keys in calls.items():
            res, nbytes = _check_call(cs, ctx, oc, [v[k] for k in keys], what=f"{name} {shape}", table=table)
            lone = [_lone_streamed(cs, v[k]) for k in keys]
            u = _union_streamed(cs, res, nbytes)
            assert max(lone) <= u <= sum(lone), (name, u, lone)
            if name == "only the masked view takes them":
                assert u == lone[0] < res[0].stats["entities_tested"], (u, lone)  # the x-index 0 pages are copied, only is_big rows read
    cs.setLaunch()
    cs.close()


def test_type_filters_mixed_with_all_types(ctx, grid):
    cs, oc, table = grid
    views = _grid_views()
    for types in ([1, ALL], [ALL, 0, 2, ALL, 1], [2, 2, 1, 0, ALL, ALL, 1, 0], [0xFF, 0xFF, 0xFF]):
        frusta = [views[i % 3] for i in range(len(types))]
        res, _ = _check_call(cs, ctx, oc, frusta, types, what=f"types {types}", table=table)
        for r, t in zip(res, types):
            if t != ALL:
                assert r.stats["pages_filtered"] > 0 and set(np.unique(r.types())) <= {t}


# ---------------------------------------------------------------- realistic frames -----------------------------------------------------

def _frame_views(cascades):
    a = scenes.c2_frustum_args()
    return [lb.frustum_perspective(**a)] + [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(a, (0.35, -0.85, 0.25), cascades)]


def test_main_view_and_cascades_on_c2(ctx, oracle):
    """The 10 M-entity C2 scene: the main view and four cascades built as prepareShadowCameras builds them, with the engine's default
    cascades and with cascades scaled to C2's far plane; then the same frame with a type filter per cascade."""
    cs, oc = _both(ctx, oracle, scenes.c2_scene())
    far = scenes.c2_frustum_args()["far"]
    for name, cascades in (("default", scenes.DEFAULT_CASCADES), ("scaled", tuple(c * far / 150.0 for c in scenes.DEFAULT_CASCADES))):
        frusta = _frame_views(cascades)
        exps = [Expect(oc, f) for f in frusta]
        assert len(exps[0].ids) and len(exps[1].ids), [len(e.ids) for e in exps]
        res, nbytes = _frame(cs, ctx, frusta)
        for v, (r, e) in enumerate(zip(res, exps)):
            _check(r, e, f"c2 {name} view {v}")
        lone = [_lone_streamed(cs, f) for f in frusta]
        u = _union_streamed(cs, res, nbytes)
        assert max(lone) <= u <= sum(lone), (name, u, lone)
        if name == "default":
            assert u < sum(lone), (u, lone)  # the near cascades lie inside the main view: their pages' rows are read once
    frusta = _frame_views(scenes.DEFAULT_CASCADES)
    types = [ALL, 0, 1, ALL, 3]
    res, _ = _frame(cs, ctx, frusta, types)
    for v, (r, f, t) in enumerate(zip(res, frusta, types)):
        _check(r, Expect(oc, f, t), f"c2 filtered view {v}")
    cs.close()


# ---------------------------------------------------------------- launch shapes ---------------------------------------------------------

def test_launch_shapes(ctx, grid):
    cs, oc, table = grid
    views = _grid_views()
    sms = _sms()
    seen = set()
    for n in (2, 5, 8):
        frusta = views[:n]
        bound = min(256, 512 // n)
        exps = [Expect(oc, f) for f in frusta]
        for blocks in (0, 1, 2, 7, sms, -1, 4000):
            for chunk in (1, 7, 31, 33, 64, 255, 0):
                what = f"{n} views blocks {blocks} chunk {chunk}"
                cs.setLaunch(blocks, chunk)
                res, _ = _frame(cs, ctx, frusta)
                for v, (r, e) in enumerate(zip(res, exps)):
                    _check(r, e, f"{what} view {v}")
                ll = cs.lastLaunch()
                if blocks > 0:
                    assert ll["blocks"] == blocks, (what, ll)
                if chunk:
                    assert ll["chunk"] == min(chunk, bound), (what, ll)
                    if chunk > bound:
                        seen.add("capped")
                b, c = ll["blocks"], ll["chunk"]
                assert 1 <= c <= bound and ll["rounds"] == -(-N_GRID_PAGES // (b * c)), (what, ll)
                if ll["rounds"] > 1:
                    seen.add("exact" if N_GRID_PAGES % (b * c) == 0 else "partial")
                if b * c > N_GRID_PAGES and b > -(-N_GRID_PAGES // c):
                    seen.add("idle blocks")
                if c < 32:
                    seen.add("chunk below a warp")
        cs.select_view(n - 1)
        assert np.array_equal(table.decode(cs.read_bitmask(), f"{n} views last shape"), exps[-1].key)
    cs.setLaunch()
    assert seen == {"capped", "exact", "partial", "idle blocks", "chunk below a warp"}, seen


# ---------------------------------------------------------------- plane masking off -----------------------------------------------------

def test_plane_masking_off(ctx, oracle):
    cs, oc = _both(ctx, oracle, _edge_scene())
    table = Table(cs)
    v = _edge_views()
    frusta = [v["copy"], v["test"], v["masked"], v["skip"]]
    cs.setLaunch(plane_masking=0)
    res, nbytes = _check_call(cs, ctx, oc, frusta, what="masking off", table=table)
    assert not cs.lastLaunch()["plane_masking"]
    tested = max(r.stats["entities_tested"] for r in res)
    assert _union_streamed(cs, res, nbytes) == tested  # every tested page is read, once: the x-index 0 pages and the is_big ones
    cs.setLaunch()
    # a negative and NaN radii of either sign switch masking off by themselves (the sign path of phase B)
    n = cs.entity_count()
    ids = np.arange(n, n + 4, dtype=np.int32)
    pos = np.array([[140.0, 100.0, 400.0], [160.0, 100.0, 700.0], [140.0, 50.0, 1000.0], [140.0, 60.0, 1300.0]])
    rad = np.array([-3.0, np.nan, -np.nan, 2.0], np.float32)
    cs.add(ids, np.zeros(4, np.uint8), pos, rad)
    oc.add(ids, np.zeros(4, np.uint8), pos, rad)
    table = Table(cs)
    for shape in ((0, 0), (3, 7)):
        cs.setLaunch(*shape)
        _check_call(cs, ctx, oc, frusta, what=f"bad radii {shape}", table=table)
        assert not cs.lastLaunch()["plane_masking"]
    cs.setLaunch()
    cs.close()


# ---------------------------------------------------------------- state and buffers ------------------------------------------------------

def test_device_authoritative_state(ctx, oracle):
    """After set_many_device, add_many_device and remove_many_device: visible sets against the oracle, statistics and mask rows against
    lone cull_device calls on the same device layout."""
    rng = np.random.default_rng(3)
    scene = scenes.cull_scene(80_000, (3000.0, 300.0, 3000.0), seed=31, big_fraction=0.003, type_probs=(0.6, 0.3, 0.1))
    cs, oc = _both(ctx, oracle, scene)
    a = scenes.c1_frustum_args()
    frusta = [lb.frustum_perspective(**dict(a, far=2500.0))] + [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(dict(a, far=2500.0), (0.3, -0.8, 0.2))]
    n = len(scene["entities"])

    def check(what):
        res, _ = _frame(cs, ctx, frusta)
        masks = []
        for v in range(len(frusta)):
            cs.select_view(v)
            masks.append(cs.read_bitmask().copy())
        for v, (f, r) in enumerate(zip(frusta, res)):
            _check(r, Expect(oc, f), f"{what} view {v}", stats=False)
            lone = ViewResult(ctx, *cs.cull_device(f))
            assert r.stats == lone.stats, (what, v, r.stats, lone.stats)
            assert np.array_equal(masks[v], cs.read_bitmask()), (what, v)

    def dev(*arrays):
        return [ctx.to_device(np.ascontiguousarray(x)) for x in arrays]

    ents = rng.choice(n, 20_000, replace=False).astype(np.int32)
    pos = scene["pos"][ents] + rng.normal(size=(len(ents), 3)) * np.array([300.0, 10.0, 300.0])
    rad = scene["radius"][ents]
    d = dev(ents, pos, rad)
    cs.set_many_device(d[1], d[2], len(ents), dev_entities=d[0], max_entity=n - 1)
    oc.set(ents, pos, rad)
    check("set_many_device")
    new = np.arange(n, n + 5000, dtype=np.int32)
    npos = (rng.random((5000, 3)) * 2 - 1) * np.array([3000.0, 300.0, 3000.0])
    nrad, nty = rng.uniform(0.5, 5.0, 5000).astype(np.float32), rng.integers(0, 3, 5000).astype(np.uint8)
    d2 = dev(new, nty, npos, nrad)
    cs.add_many_device(d2[2], d2[3], d2[1], len(new), dev_entities=d2[0], max_entity=n + 4999)
    oc.add(new, nty, npos, nrad)
    check("add_many_device")
    gone = rng.choice(n, 7000, replace=False).astype(np.int32)
    d3 = dev(gone)
    cs.remove_many_device(d3[0], len(gone))
    oc.remove(gone)
    check("remove_many_device")
    for p in d + d2 + d3:
        ctx.free_device(p)
    cs.close()


def test_replicas_rotate(ctx, oracle):
    scene = scenes.cull_scene(60_000, (3000.0, 300.0, 3000.0), seed=61, big_fraction=0.01, type_probs=(0.5, 0.3, 0.2))
    cs, oc = _both(ctx, oracle, scene)
    cs.set_replicas(3)
    views = _c1_views()
    table = Table(cs)
    for i in range(5):  # five calls over three replicas, each with its own view set
        frusta = views[i % 3:i % 3 + 4]
        _check_call(cs, ctx, oc, frusta, what=f"replicas call {i}", table=table)
        cs.setPosition(scene["entities"][i * 10:i * 10 + 5], scene["pos"][i * 10:i * 10 + 5] + 40.0)
        oc.set_position(scene["entities"][i * 10:i * 10 + 5], scene["pos"][i * 10:i * 10 + 5] + 40.0)
        table = Table(cs)
    cs.close()


def test_entity_growth_and_page_growth(ctx, oracle):
    scene = scenes.cull_scene(3000, (2000.0, 200.0, 2000.0), seed=5, type_probs=(0.5, 0.5))
    cs, oc = _both(ctx, oracle, scene)
    frusta = _c1_views()[:5]
    _check_call(cs, ctx, oc, frusta, what="before growth")
    # more entities than the view id buffers hold, in the same region: the buffers grow at the next call
    more = scenes.cull_scene(30_000, (2000.0, 200.0, 2000.0), seed=6, type_probs=(0.5, 0.5))
    ids = more["entities"] + 3000
    cs.add(ids, more["types"], more["pos"], more["radius"])
    oc.add(ids, more["types"], more["pos"], more["radius"])
    _check_call(cs, ctx, oc, frusta, what="after entity growth")
    cs.select_view(2)
    # a growth of the page arrays releases the view buffers: select_view refuses, last_result too
    far = scenes.cull_scene(30_000, (20000.0, 200.0, 20000.0), seed=7)
    cs.add(far["entities"] + 40_000, far["types"], far["pos"], far["radius"])
    oc.add(far["entities"] + 40_000, far["types"], far["pos"], far["radius"])
    cs.flush()
    for k in (0, 4):
        with pytest.raises(lb.LumixB200Error) as e:
            cs.select_view(k)
        assert e.value.code == _lib.ERR_STATE
    with pytest.raises(lb.LumixB200Error) as e:
        cs.last_result()
    assert e.value.code == _lib.ERR_STATE
    _check_call(cs, ctx, oc, frusta, what="after page growth")
    cs.set_replicas(2)
    with pytest.raises(lb.LumixB200Error) as e:
        cs.select_view(0)
    assert e.value.code == _lib.ERR_STATE
    cs.close()


def test_independent_of_the_lanes(ctx, c1):
    """A cull_device pointer and its result survive a cull_views call, and the view buffers survive plain culls on every lane."""
    cs, oc, table = c1
    views = _c1_views()
    e0 = Expect(oc, views[6])
    ptr, raw = cs.cull_device(views[6])
    seq_launch = ctx.launches
    res, _ = _frame(cs, ctx, views[:5])
    assert ctx.launches == seq_launch + 1  # one fused launch for five views
    _check(ViewResult(ctx, ptr, raw), e0, "cull_device after cull_views")
    lp, lr = cs.last_result()
    assert lp == ptr and int(lr.total) == len(e0.ids)
    out = cs.cull_views(views[:5])
    for _ in range(8):
        cs.cull_device(views[7], want_counts=False)
    cs.cull_device_n(views[6], 4)
    for v, (p, r) in enumerate(out):
        e = Expect(oc, views[v])
        _check(ViewResult(ctx, p, r), e, f"view {v} after plain culls")
        cs.select_view(v)
        assert np.array_equal(table.decode(cs.read_bitmask(), f"view {v} after plain culls"), e.key)
        lp, lr = cs.last_result()
        assert lp == p and int(lr.total) == len(e.ids)


# ---------------------------------------------------------------- createSortKeys per view ----------------------------------------------

def test_sort_keys_per_view(ctx, oracle):
    n = 60_000
    scene = scenes.cull_scene(n, (2500.0, 300.0, 2500.0), seed=11, type_probs=(0.8, 0.08, 0.04, 0.08), big_fraction=0.002)
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=111)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setTransforms(sk["transforms"])
    a = dict(scenes.c1_frustum_args(), far=2500.0)
    frusta = [lb.frustum_perspective(**a)] + [lb.frustum_ortho(**s) for s in scenes.shadow_cascade_args(a, (0.3, -0.8, 0.2), (40.0, 200.0, 900.0, 2500.0))]
    cs.cull_views(frusta, want_counts=False)

    def keys(view):
        S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])  # same lod / pose state
        res = S.createSortKeys(cs, view)
        return res, S.read(res)

    for k, f in enumerate(frusta):
        view = sortkeys.make_view(a["position"], a["position"], 1.0 / 30.0, 1.0, 50, k > 0, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
        cs.select_view(k)
        r1, got = keys(view)
        cs.cull_device(f, want_counts=False)
        r2, exp = keys(view)
        assert r1.n_keys == r2.n_keys and r1.n_instances == r2.n_instances, (k, r1.n_keys, r2.n_keys)
        assert r1.n_keys > 0 or k > 0
        gk = np.lexsort((got["values"], got["keys"]))
        ek = np.lexsort((exp["values"], exp["keys"]))
        assert np.array_equal(got["keys"][gk], exp["keys"][ek]) and np.array_equal(got["values"][gk], exp["values"][ek]), k
        assert np.array_equal(got["group_count"], exp["group_count"]) and np.array_equal(got["group_offset"], exp["group_offset"]), k
        go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
        assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo]), k
        assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo]), k
    S.close()
    cs.close()


# ---------------------------------------------------------------- refusals --------------------------------------------------------------

def test_refusals(ctx, c1):
    cs, oc, _ = c1
    L = cs.L
    f = _c1_views()[0]
    arr = (_lib.ShiftedFrustum * 9)(*([f] * 9))
    ids = (C.c_void_p * 9)()
    res = (_lib.CullResult * 9)()
    for frusta, n in ((arr, 0), (arr, 9), (None, 2), (None, 0)):
        assert L.lb200_culling_cull_views(cs.h, frusta, None, C.c_uint32(n), ids, res, C.c_int(1)) == _lib.ERR_INVALID, n
    cs.cull_views([f, f])
    for k in (2, 8, 1 << 31):
        with pytest.raises(lb.LumixB200Error) as e:
            cs.select_view(k)
        assert e.value.code == _lib.ERR_INVALID
    fresh = lb.CullingSystem(ctx)
    with pytest.raises(lb.LumixB200Error) as e:
        fresh.select_view(0)
    assert e.value.code == _lib.ERR_STATE
    # an empty culling system: zero results, nothing launched, nothing to select
    before = ctx.launches
    out = fresh.cull_views([f] * 5)
    assert ctx.launches == before and all(p == 0 and r.total == 0 and r.pages_outside == 0 for p, r in out)
    with pytest.raises(lb.LumixB200Error) as e:
        fresh.select_view(0)
    assert e.value.code == _lib.ERR_STATE
    assert L.lb200_culling_cull_views(fresh.h, arr, None, C.c_uint32(0), ids, res, C.c_int(1)) == _lib.ERR_INVALID
    fresh.close()
