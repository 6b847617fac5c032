"""cull_pages_kernel at every launch shape, held to the oracle.

launchCull picks the grid and the pages per block per round (chunk) from the page count: chunk = ceil(pages / resident blocks) within
32..256, and never more blocks than are co-resident.  So a cull runs a second round only beyond 256 pages per resident block (135,168
pages for a plain cull on a 132-SM H100, half that on a lane), and the classify pass always has at least a warp of page slots.
CullingSystem.setLaunch forces the grid (1, 2, 3, 7, one and two blocks per SM, every co-resident block, more blocks than fit and than
there are pages) and the chunk (1..256), so that the round loop, exactly and partly full last rounds, blocks without a page and chunks
below a warp run on scenes of a few thousand pages.  Every cull is compared with oracle.OracleCulling on the same edits: the visible set
per renderable type, the six statistics, and the visibility rows of the mask decoded through the page table.
"""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib

pytestmark = pytest.mark.gpu

STATS = ("pages_tested", "pages_inside", "pages_outside", "pages_filtered", "entities_tested", "entities_inside")
CELL = 300.0
CHUNKS = (1, 7, 31, 32, 33, 64, 128, 255, 256, 0)
SENTINEL = 0xDEADBEEF


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Expect:
    """The oracle's answer for one (scene, view, type): it does not depend on the launch shape."""

    def __init__(self, oc, f, type=-1):
        self.ids, self.tys, self.st = oc.cull(lb.culling.frustum_bytes(f), type)
        self.key = np.sort(self.ids.astype(np.int64) * 256 + self.tys)


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


def _check_mask(cs, table, exp, what):
    bits = np.unpackbits(cs.read_bitmask().view(np.uint8), bitorder="little").reshape(-1, 256).astype(bool)
    assert not (bits & ~table.live).any(), f"{what}: mask bits at or beyond a page's count"
    got = np.sort(table.ent[bits] * 256 + np.broadcast_to(table.type[:, None], bits.shape)[bits])
    assert np.array_equal(got, exp.key), f"{what}: mask rows decode to {int(bits.sum())} ids, oracle {len(exp.ids)}"


def _streamed(cs, res):
    """Spheres the last cull read, from its algorithmic bytes (64 B per page + 16 B per streamed sphere + 8 B per visible id);
    valid while the page high-water mark is the page count (no page was freed)."""
    rest = cs.last_algorithmic_bytes() - 64 * cs.page_count() - 8 * res.total
    assert rest >= 0 and rest % 16 == 0
    return rest // 16


def _x_cut(x, inside_below, cz=0.0, extent=6000.0):
    """Ortho view whose inside is x <= x (inside_below) or x >= x, `extent` wide in x and z (around cz), y in +-5000 (computeOrtho takes
    half sizes; this camera faces -y, so the volume runs from the near plane at y = -5000 up to the far plane)."""
    px = x - extent / 2 if inside_below else x + extent / 2
    for _ in range(4):
        f = lb.frustum_ortho((px, -5000.0, cz), (0.0, -1.0, 0.0), (0.0, 0.0, 1.0), extent / 2, extent / 2, 0.0, 10000.0)
        i = [p for p in range(6) if (f.xs[p] < -0.99 if inside_below else f.xs[p] > 0.99)]
        assert len(i) == 1
        edge = f.origin[0] + f.ds[i[0]] if inside_below else f.origin[0] - f.ds[i[0]]  # inside: n . (p - origin) + d >= 0
        if abs(edge - x) < 1e-3:
            return f
        px += x - edge
    raise AssertionError(f"ortho view edge at {edge}, wanted {x}")


# ---------------------------------------------------------------- the launch-shape sweep ----------------------------------------------

N_GRID_PAGES = 3584  # 2^9 x 7: the last round is exactly full at 1, 2 and 7 blocks with chunks 1, 7, 32, 64, 128 and 256


def _grid_scene(seed=7):
    """1,792 cells (32 in x by 56 in z, one layer) with two pages each, of different renderable types: 3,584 pages of 1..40 entities
    (every fourth cell 1..200), the second page of every 17th cell is_big."""
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
    # across the grid from its -z edge: pages inside (shifted box contained), pages tested and pages outside
    a = lb.frustum_perspective((5100.0, 150.0, -200.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 1.2, 1.0, 0.5, 9000.0)
    nothing = lb.frustum_perspective((1e6, 0.0, 1e6), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 1.2, 1.0, 0.5, 100.0)
    return {"all": (a, lb.culling.TYPE_ALL), "type1": (a, 1), "nothing": (nothing, lb.culling.TYPE_ALL)}


@pytest.fixture(scope="module")
def grid(ctx, oracle):
    scene = _grid_scene()
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    assert cs.page_count() == oc.page_count() == N_GRID_PAGES
    yield cs, oc, Table(cs)
    cs.close()


@pytest.mark.parametrize("view", ["all", "type1", "nothing"])
def test_every_shape_with_and_without_plane_masking(grid, view):
    cs, oc, table = grid
    f, t = _grid_views()[view]
    exp = Expect(oc, f, -1 if t == lb.culling.TYPE_ALL else t)
    if view == "all":
        assert exp.st["pages_tested"] and exp.st["pages_inside"] and exp.st["pages_outside"] and len(exp.ids), exp.st
    if view == "type1":
        assert exp.st["pages_filtered"] and len(exp.ids), exp.st
    if view == "nothing":
        assert len(exp.ids) == 0 and exp.st["pages_inside"] == 0 and exp.st["pages_tested"], exp.st  # is_big pages are always tested
    sms = _sms()
    seen = set()
    for blocks in (0, 1, 2, 3, 7, sms, 2 * sms, -1, 4000):
        for chunk in CHUNKS:
            what = f"{view} blocks {blocks} chunk {chunk}"
            cs.setLaunch(blocks, chunk)
            on = cs.cull(f, t)
            _check(on, exp, what)
            _check_mask(cs, table, exp, what)
            ll = cs.lastLaunch()
            s_on = _streamed(cs, on)
            assert ll["plane_masking"], what
            if blocks > 0:
                assert ll["blocks"] == blocks, what
            if chunk:
                assert ll["chunk"] == chunk, what
            b, c = ll["blocks"], ll["chunk"]
            assert 1 <= c <= 256 and ll["rounds"] == -(-N_GRID_PAGES // (b * c)), (what, ll)
            if ll["rounds"] > 1:
                seen.add("exact" if N_GRID_PAGES % (b * c) == 0 else "partial")
            seen.add("one round" if ll["rounds"] == 1 else "rounds")
            if b > N_GRID_PAGES:
                seen.add("idle blocks")
            if c < 32:
                seen.add("chunk below a warp")
            cs.setLaunch(blocks, chunk, plane_masking=0)
            off = cs.cull(f, t)
            _check(off, exp, what + " masking off")
            _check_mask(cs, table, exp, what + " masking off")
            assert not cs.lastLaunch()["plane_masking"], what
            assert _streamed(cs, off) >= s_on, what
            assert _streamed(cs, off) == exp.st["entities_tested"], what  # without masking every tested page is read
    cs.setLaunch()
    assert seen == {"one round", "rounds", "exact", "partial", "idle blocks", "chunk below a warp"}, seen


def test_set_launch_rejects_other_values(ctx):
    cs = lb.CullingSystem(ctx)
    assert cs.lastLaunch() == dict(blocks=0, chunk=0, rounds=0, pdl=False, plane_masking=False)
    for blocks, chunk, masking in ((-2, 0, -1), (0, -1, -1), (0, 257, -1), (0, 0, 1), (0, 0, -2), ((1 << 20) + 1, 0, -1)):
        with pytest.raises(lb.LumixB200Error) as e:
            cs.setLaunch(blocks, chunk, masking)
        assert e.value.code == _lib.ERR_INVALID
    cs.setLaunch(1 << 20, 256, 0)
    cs.setLaunch(-1, 1, -1)
    cs.close()


# ---------------------------------------------------------------- the default rule beyond one round ----------------------------------

def test_default_rule_goes_multi_round(ctx, oracle):
    """A sparse open world of 140,000 occupied cells, one entity each: beyond 256 pages per co-resident block of a plain cull on a
    132-SM H100 (135,168) and of a lane (67,584), so the default rule itself runs more than one round.  Footprint: about 0.6 GB of page
    arrays on the device (4 KB per page) and the same in page-locked host memory."""
    n_x, n_z = 400, 350
    i, j = np.meshgrid(np.arange(n_x), np.arange(n_z), indexing="ij")
    i, j = i.ravel(), j.ravel()
    pos = np.stack([i * CELL + 150.0, np.full(i.shape, 150.0), j * CELL + 150.0], 1)
    scene = dict(entities=np.arange(len(pos), dtype=np.int32), types=((i + j) % 3).astype(np.uint8), pos=pos,
                 radius=np.full(len(pos), 2.0, np.float32))
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    n_pages = cs.page_count()
    assert n_pages == n_x * n_z
    f = lb.frustum_perspective((30000.0, 400.0, -500.0), (0.2, -0.05, 1.0), (0.0, 1.0, 0.0), 1.3, 1.6, 0.5, 80000.0)
    exp = Expect(oc, f)
    assert exp.st["pages_tested"] and exp.st["pages_inside"] and exp.st["pages_outside"], exp.st
    res = cs.cull(f)
    _check(res, exp, "plain cull")
    ll = cs.lastLaunch()
    assert ll["chunk"] == 256 and ll["rounds"] == 2, ll
    assert int(np.unpackbits(cs.read_bitmask().view(np.uint8)).sum()) == len(exp.ids)
    cs.cull_device_n(f, 4)
    ptr, last = cs.last_result()
    ll = cs.lastLaunch()
    assert ll["chunk"] == 256 and ll["rounds"] > 1 and ll["rounds"] == -(-n_pages // (ll["blocks"] * 256)), ll
    assert ll["blocks"] * 256 < n_pages, ll
    base = np.concatenate([[0], np.cumsum(np.bincount(scene["types"], minlength=256))])
    for t in range(3):
        got = ctx.copy_to_host(ptr + 4 * int(base[t]), int(last.type_count[t]), np.uint32)
        assert np.array_equal(np.sort(got).astype(np.int64), np.sort(exp.ids[exp.tys == t]).astype(np.int64)), t
    for k in STATS:
        assert getattr(last, k) == exp.st[k], k
    assert int(np.unpackbits(cs.read_bitmask().view(np.uint8)).sum()) == len(exp.ids)
    cs.close()


# ---------------------------------------------------------------- page-count edges --------------------------------------------------

EDGE_COUNTS = (1, 31, 32, 33, 127, 128, 129, 160, 199, 200, 201, 400)
EDGE_SHAPES = ((0, 0), (1, 1), (1, 7), (2, 31), (3, 32), (7, 33), (-1, 0), (1000, 1), (2, 256))


def _visible_slot(pattern, s, n):
    return (s % 2 == 0, s == n - 1, s == 128, s % 3 != 0)[pattern]


def _edge_scene():
    """One cell per count in EDGE_COUNTS at x-index 0 (x in [0, 300)), one after another in z, renderable type = cell % 3.  Slot s of a
    cell (insertion order) lies 20 m left of the plane x = 150 (visible in the cut view) or 20 m right of it, by the cell's pattern:
    alternating, the last slot only, slot 128 only, or every slot but each third.  Two is_big cells (129 and 200 spheres of radius
    301..400) at x-index 1."""
    rng = np.random.default_rng(17)
    tys, pos, rad = [], [], []
    for k, n in enumerate(EDGE_COUNTS):
        vis = np.array([_visible_slot(k % 4, s, n) for s in range(n)])
        x = np.where(vis, 130.0, 170.0)
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


def _edge_views():
    cz = (len(EDGE_COUNTS) + 2) * CELL / 2
    return {"test": _x_cut(150.0, True, cz),   # cuts every cell: TEST pages
            "copy": _x_cut(1000.0, True, cz),  # holds the shifted box [origin + 300, origin + 600] of x-index 0: COPY pages
            "masked": _x_cut(450.0, True, cz)}  # holds the cells, not their shifted boxes: TEST pages that plane masking copies


def _edge_system(ctx, oracle):
    scene = _edge_scene()
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    table = Table(cs)
    counts = sorted(int(c) for c in table.count)
    assert counts == sorted([1, 31, 32, 33, 127, 128, 129, 160, 199, 200, 200, 1, 200, 200, 129, 200]), counts
    return cs, oc, table, scene


def test_page_count_edges(ctx, oracle):
    cs, oc, table, _ = _edge_system(ctx, oracle)
    n_pages = cs.page_count()
    classes = set()
    for name, f in _edge_views().items():
        exp = Expect(oc, f)
        if name == "test":
            assert exp.st["pages_tested"] == n_pages and exp.st["pages_inside"] == 0, exp.st
        if name == "copy":
            assert exp.st["pages_inside"] == n_pages - 2 and exp.st["pages_tested"] == 2, exp.st
        if name == "masked":
            assert exp.st["pages_tested"] == n_pages and exp.st["pages_inside"] == 0, exp.st
        for blocks, chunk in EDGE_SHAPES:
            what = f"{name} blocks {blocks} chunk {chunk}"
            cs.setLaunch(blocks, chunk)
            res = cs.cull(f)
            _check(res, exp, what)
            _check_mask(cs, table, exp, what)
            s_on = _streamed(cs, res)
            cs.setLaunch(blocks, chunk, plane_masking=0)
            off = cs.cull(f)
            _check(off, exp, what + " masking off")
            _check_mask(cs, table, exp, what + " masking off")
            s_off = _streamed(cs, off)
            assert s_off == res.stats["entities_tested"] and s_on <= s_off, what
            if res.stats["pages_inside"]:
                classes.add("copy")
            if s_on:
                classes.add("test")
            if s_on < res.stats["entities_tested"]:
                classes.add("masked")  # the cells lie inside every plane: in the copy view that holds for the is_big pages too
            if name == "test":
                assert s_on == res.stats["entities_tested"], what
            if name == "masked":
                assert s_on < res.stats["entities_tested"], what
    assert classes == {"copy", "test", "masked"}, classes
    cs.setLaunch()
    cs.close()


# ---------------------------------------------------------------- mask rows across culls on one lane ----------------------------------

def test_mask_rows_of_pages_skipped_after_work(ctx, oracle):
    """A lane's mask buffer is reused by every later cull on it.  View A works the pages of x-index 0; view B has its plane 0.01 m beyond
    their intersects box (x <= 300), inside the cheap pass's 0.05 m margin, so only the exact pass skips them and has to zero their
    rows.  A is culled eight times first (as many as there can be lanes), so that B lands on a lane whose rows are A's."""
    cs, oc, table, scene = _edge_system(ctx, oracle)
    a = _edge_views()["test"]
    b = _x_cut(300.01, False, (len(EDGE_COUNTS) + 2) * CELL / 2)
    ea, eb = Expect(oc, a), Expect(oc, b)
    assert len(ea.ids) and eb.st["pages_tested"] == 2 and eb.st["pages_outside"] == cs.page_count() - 2, eb.st
    for blocks, chunk in ((0, 0), (1, 7), (3, 1)):
        cs.setLaunch(blocks, chunk)
        for _ in range(8):
            _check(cs.cull(a), ea, f"A blocks {blocks} chunk {chunk}")
        _check_mask(cs, table, ea, f"A blocks {blocks} chunk {chunk}")
        _check(cs.cull(b), eb, f"B blocks {blocks} chunk {chunk}")
        _check_mask(cs, table, eb, f"B blocks {blocks} chunk {chunk}")
        if (blocks, chunk) != (0, 0):
            assert cs.lastLaunch()["rounds"] > 1
    # a freed page gets a zero row: empty the 33-entity cell (it has visible slots in A), cull A on every lane, then reuse the page for
    # a new cell without culling: read_bitmask shows the row the last cull wrote for it while it was free
    k = EDGE_COUNTS.index(33)
    pages = cs.pages()
    victim = [i for i, p in enumerate(pages) if p["count"] == 33][0]
    freed = int(cs.page_ids()[victim])
    gone = pages[victim]["entities"]
    cs.remove(gone)
    oc.remove(gone)
    ea = Expect(oc, a)
    cs.setLaunch(1, 7)
    for _ in range(8):
        _check(cs.cull(a), ea, "A after the removal", stats=True)
    new_id = int(scene["entities"].max()) + 1
    cs.add(new_id, 0, (140.0, 100.0, 40 * CELL + 100.0), 2.0)
    ids = cs.page_ids()
    assert freed in ids, "the new cell did not take the freed page"
    row = cs.read_bitmask()[int(np.nonzero(ids == freed)[0][0])]
    assert not row.any(), f"the freed page {freed} (cell {k}) kept the row {row}"
    cs.setLaunch()
    cs.close()


# ---------------------------------------------------------------- programmatic dependent launch ------------------------------------

def test_pdl_at_changing_shapes(ctx, oracle):
    cs, oc, table, scene = _edge_system(ctx, oracle)
    views = _edge_views()
    exps = {k: Expect(oc, f) for k, f in views.items()}
    seen = set()
    for edit in range(3):
        if edit:
            e = scene["entities"][edit * 7:edit * 7 + 3]
            p = scene["pos"][edit * 7:edit * 7 + 3] + np.array([0.0, 0.0, 3.0])
            cs.setPosition(e, p)
            oc.set_position(e, p)
            exps = {k: Expect(oc, f) for k, f in views.items()}
        for i, (blocks, chunk) in enumerate(EDGE_SHAPES):
            name = ("test", "copy", "masked")[i % 3]
            cs.setLaunch(blocks, chunk)
            res = cs.cull(views[name])
            _check(res, exps[name], f"edit {edit} {name} blocks {blocks} chunk {chunk}")
            pdl = cs.lastLaunch()["pdl"]
            assert pdl == (i > 0), (edit, i, pdl)  # the first cull after an upload is launched plain
            seen.add(pdl)
    assert seen == {True, False}
    cs.setLaunch()
    cs.close()


# ---------------------------------------------------------------- replicas ---------------------------------------------------------

def test_replicas_round_robin(ctx, oracle):
    from lumixengine_b200 import scenes
    scene = scenes.cull_scene(60_000, (3000.0, 300.0, 3000.0), seed=61, big_fraction=0.01, type_probs=(0.5, 0.3, 0.2))
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    cs.set_replicas(3)
    a = scenes.c1_frustum_args()
    views = [lb.frustum_perspective(**dict(a, far=2500.0)),
             lb.frustum_perspective(**dict(a, position=(800.0, 0.0, 900.0), direction=(-0.5, 0.0, -0.8), far=1700.0)),
             lb.frustum_ortho((0.0, 0.0, 4000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 3000.0, 3000.0, 0.0, 8000.0)]
    pos = scene["pos"].copy()
    rng = np.random.default_rng(5)

    def culls(n, what):
        exps = [Expect(oc, f) for f in views]
        for i in range(n):  # views and replicas rotate at the same period: shift the view every third cull
            v = (i + i // 3) % 3
            _check(cs.cull(views[v]), exps[v], f"{what} cull {i}")

    def move(n):
        e = rng.choice(len(pos), n, replace=False).astype(np.int32)
        pos[e] += rng.normal(size=(n, 3)) * np.array([200.0, 20.0, 200.0])
        cs.setPosition(e, pos[e])
        oc.set_position(e, pos[e])

    for blocks, chunk in ((0, 0), (3, 7)):
        cs.setLaunch(blocks, chunk)
        culls(7, f"blocks {blocks}")
        move(20)  # a sparse upload: scattered into every replica
        culls(3, f"blocks {blocks} after a sparse upload")
        move(30_000)  # a full upload
        culls(3, f"blocks {blocks} after a full upload")
    assert cs.lastLaunch()["rounds"] > 1
    cs.setLaunch()
    ents = np.arange(0, len(pos), 7, dtype=np.int32)
    new_pos = pos[ents] + np.array([35.0, 0.0, -50.0])
    new_rad = scene["radius"][ents]
    d_e, d_p, d_r = ctx.to_device(ents), ctx.to_device(np.ascontiguousarray(new_pos)), ctx.to_device(new_rad)
    try:
        with pytest.raises(lb.LumixB200Error) as e:
            cs.set_many_device(d_p, d_r, len(ents), dev_entities=d_e, max_entity=len(pos) - 1)
        assert e.value.code == _lib.ERR_STATE
        cs.set_replicas(1)
        cs.set_many_device(d_p, d_r, len(ents), dev_entities=d_e, max_entity=len(pos) - 1)
        oc.set(ents, new_pos, new_rad)
        for f in views:
            exp = Expect(oc, f)
            res = cs.cull(f)
            _check(res, exp, "after device re-binning", stats=False)  # device re-binning places pages differently by design
    finally:
        for p in (d_e, d_p, d_r):
            ctx.free_device(p)
    cs.close()


# ---------------------------------------------------------------- exchange at multi-round shapes -------------------------------------

def test_exchange_one_rank_at_multi_round_shapes(oracle):
    """The cull kernel's exchange mode ({page, row} records and per-type counts stored into every rank's slab) with a world of one
    rank, in its own context: single steps and fused batches on the lanes, at the default shape and at shapes of several rounds."""
    from lumixengine_b200 import scenes
    ctx = lb.Context(0)
    try:
        ctx.comm_init(1, 0, ctx.comm_unique_id())
        scene = scenes.cull_scene(80_000, (3000.0, 300.0, 3000.0), seed=71, big_fraction=0.004, type_probs=(0.6, 0.3, 0.1))
        cs = lb.CullingSystem(ctx)
        cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
        oc = oracle.OracleCulling()
        oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
        ctx.comm_enable_p2p(cs.exchange_slab_words() - 256)
        table, pid = Table(cs), cs.page_ids()
        base = np.concatenate([[0], np.cumsum(np.bincount(scene["types"], minlength=256))])
        a = scenes.c1_frustum_args()
        views = [lb.frustum_perspective(**dict(a, far=2500.0)),
                 lb.frustum_perspective(position=(500.0, 20.0, -300.0), direction=(0.6, -0.1, 0.79), up=(0, 1, 0), fov=0.9, ratio=1.6, near=0.5, far=1800.0)]
        exps = [Expect(oc, f) for f in views]
        for blocks, chunk in ((0, 0), (1, 7), (3, 33), (-1, 1), (1000, 256)):
            cs.setLaunch(blocks, chunk)
            for step in range(3):
                v = step % 2
                what = f"blocks {blocks} chunk {chunk} step {step}"
                if step == 2:
                    ids_ptr, slabs_ptr, stride = cs.cull_exchange_n(views[v], 5)
                else:
                    ids_ptr, slabs_ptr, stride = cs.cull_exchange(views[v])
                got = cs.read_exchanged(slabs_ptr, stride, 1)[0]
                exp = exps[v]
                for t in range(3):
                    assert int(got["counts"][t]) == int((exp.tys == t).sum()), (what, t)
                assert got["n_pages"] == int(pid.max()) + 1, what
                bits = np.unpackbits(got["mask"][pid].view(np.uint8), bitorder="little").reshape(-1, 256).astype(bool)
                assert not (bits & ~table.live).any(), what
                decoded = np.sort(table.ent[bits] * 256 + np.broadcast_to(table.type[:, None], bits.shape)[bits])
                assert np.array_equal(decoded, exp.key), what
                mine = np.concatenate([ctx.copy_to_host(ids_ptr + 4 * int(base[t]), int(got["counts"][t]), np.uint32) for t in range(3)])
                assert np.array_equal(np.sort(mine).astype(np.int64), np.sort(exp.ids).astype(np.int64)), what
                if blocks in (1, 3, -1):
                    assert cs.lastLaunch()["rounds"] > 1, what
        cs.close()
    finally:
        ctx.close()


# ---------------------------------------------------------------- pinned capacity edges -------------------------------------------

def test_pinned_capacity_edges(ctx, oracle):
    """lb200_culling_cull and cull_begin / cull_end into page-locked memory: a capacity equal to the visible count succeeds; one id less
    is LB200_ERR_CAPACITY with the total still reported, and no word at or past the capacity is written."""
    cs, oc, table, _ = _edge_system(ctx, oracle)
    f = _edge_views()["test"]
    exp = Expect(oc, f)
    total = len(exp.ids)
    buf = ctx.host_alloc(total + 256, np.uint32)
    res = _lib.CullResult()
    L = cs.L
    for blocks, chunk in ((0, 0), (3, 7), (1000, 1)):
        cs.setLaunch(blocks, chunk)
        for cap, want in ((total, _lib.OK), (total - 1, _lib.ERR_CAPACITY)):
            for how in ("cull", "begin/end"):
                what = f"{how} blocks {blocks} chunk {chunk} capacity {cap}"
                buf[:] = SENTINEL
                if how == "cull":
                    rc = L.lb200_culling_cull(cs.h, C.byref(f), C.c_uint8(0xFF), buf.ctypes.data_as(C.c_void_p), C.c_uint32(cap), C.byref(res))
                else:
                    assert L.lb200_culling_cull_begin(cs.h, C.byref(f), C.c_uint8(0xFF), buf.ctypes.data_as(C.c_void_p), C.c_uint32(cap)) == _lib.OK
                    rc = L.lb200_culling_cull_end(cs.h, C.byref(res))
                assert rc == want and res.total == total, (what, rc, res.total)
                assert (buf[cap:] == SENTINEL).all(), f"{what}: words at or past the capacity written"
                if want == _lib.OK:
                    got = np.concatenate([np.sort(buf[res.type_offset[t]:res.type_offset[t] + res.type_count[t]]).astype(np.int64) * 256 + t for t in range(3)])
                    assert np.array_equal(np.sort(got), exp.key), what
    cs.setLaunch()
    cs.close()
