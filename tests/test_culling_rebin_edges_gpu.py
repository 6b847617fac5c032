"""Device re-binning (set_many_device, add_many_device, remove_many_device, csrc/culling_rebin.cu) at the edges of its cell grid, its types
and its batch sizes, against the oracle's sequential CullingSystem::add / remove / set: the same visible sets per type over perspective
and ortho views placed where the edits are, a pulled-back mirror that holds every live entity in the cell trunc(pos * f64(f32(1 / 300)))
with its exact sphere, and set_many_device's changer count equal to the movers whose cell or is_big changed.

The device keys a chain by 18 bits per cell axis: cells [-131 072, 131 071] stay on the device, a batch that reaches further is applied
by the host bookkeeping, so two chains 262 144 cells apart never share a key."""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys
from test_culling_device_edits_gpu import Twin, _bits, _canon

pytestmark = pytest.mark.gpu

INV = np.float64(np.float32(1 / 300.0))  # IVec3(pos * (1 / 300.f)): DVec3 * float
KEY_LO, KEY_HI = -131_072, 131_071       # the cells the packed device key holds
ALIAS = 262_144                          # cells apart on one axis: the same 18 key bits


def _cells(pos):
    return np.trunc(np.asarray(pos, np.float64) * INV).astype(np.int64)


def _in_cell(rng, cell, k, margin=20.0):
    """k positions strictly inside `cell` (trunc toward zero: a negative cell c spans (300c - 300, 300c])."""
    cell = np.asarray(cell, np.float64)
    u = margin + (300.0 - 2 * margin) * rng.random((k, 3))
    pos = np.where(cell >= 0, cell * 300.0 + u, cell * 300.0 - u)
    assert (_cells(pos) == cell.astype(np.int64)).all()
    return pos


def _views_at(center, half=3000.0):
    c = np.asarray(center, np.float64)
    a = scenes.c1_frustum_args()
    return [lb.frustum_perspective(**dict(a, position=tuple(c + [0.0, 0.0, 0.5 * half]), far=1.5 * half)),
            lb.frustum_perspective(**dict(a, position=tuple(c + [0.7 * half, 20.0, -0.4 * half]), direction=(-0.7, -0.05, 0.7), far=1.5 * half)),
            lb.frustum_ortho(tuple(c + [0.0, 0.0, half]), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), half, half, 0.0, 2 * half)]


class Edge(Twin):
    """Twin whose set_many_device batches must return the exact changer count, with launch counting and mask / statistics checks."""

    def expected_changers(self, ids, pos, rad):
        ids = np.asarray(ids, np.int64)
        moved = np.any(_cells(self.pos[ids]) != _cells(pos), axis=1) | ((self.rad[ids] > 300.0) != (np.asarray(rad, np.float32) > 300.0))
        return int((moved & self.alive[ids]).sum())

    def set(self, ids, pos, rad, max_entity, what=""):
        ids, pos, rad = np.asarray(ids, np.int32), np.asarray(pos, np.float64), np.asarray(rad, np.float32)
        exp = self.expected_changers(ids, pos, rad)
        d = self._dev(ids, pos, rad)
        got = self.cs.set_many_device(d[1], d[2], len(ids), dev_entities=d[0], max_entity=max_entity)
        self._free(d)
        self.oc.set(ids, pos, rad)
        self.pos[ids], self.rad[ids] = pos, rad
        assert got == exp, f"{what}: set_many_device reports {got} changers, {exp} movers changed cell or is_big"
        return got

    def launches(self, fn, *args, **kw):
        before = self.ctx.launches
        fn(*args, **kw)
        return self.ctx.launches - before

    def check(self, what, mirror=True):
        self.check_culls(what)
        if mirror:
            self.check_mirror()

    def check_mask_and_stats(self, f, what):
        """read_bitmask decoded through the pulled-back page table equals the cull's ids; every non-empty page is counted once."""
        res = self.cs.cull(f)
        ids = np.sort(res.ids.astype(np.int64))
        st = dict(res.stats)
        pages = self.cs.pages()
        bits = np.unpackbits(self.cs.read_bitmask().view(np.uint8), bitorder="little").reshape(-1, 256).astype(bool)
        assert len(bits) == len(pages)
        for i, p in enumerate(pages):
            assert not bits[i, p["count"]:].any(), f"{what}: mask bits at or beyond the count of page {i}"
        got = np.concatenate([p["entities"][bits[i, :p["count"]]] for i, p in enumerate(pages)] + [np.zeros(0, np.int32)])
        assert np.array_equal(np.sort(got.astype(np.int64)), ids), f"{what}: mask rows"
        assert st["pages_tested"] + st["pages_inside"] + st["pages_outside"] + st["pages_filtered"] == len(pages), (what, st, len(pages))


def _ulps(x, k):
    """x and its k neighbours on either side (doubles)."""
    out = [x]
    lo = hi = x
    for _ in range(k):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [lo, hi]
    return out


def _border_positions(rng):
    """Per axis value sets: cell 0 inside (-300, 300), +-300 and other exact multiples of 300 (negative ones too), and a few ulps either
    side of the points where trunc(p * f64(f32(1/300))) and trunc(p / 300) disagree, for cells up to +-1e5."""
    vals = [-299.0, -10.0, -0.0, 0.0, 10.0, 299.0]
    for k in (1, -1, 2, -2, 7, -7, 1000, -1000):
        vals += _ulps(300.0 * k, 2)
    disagree = []
    for k in (1, -1, 3, -3, 77, -77, 4096, -4096, 33_333, -33_333, 99_999, -99_999, 100_000, -100_000):
        b = k / INV  # trunc(p * INV) reaches k here (INV > 1/300): just below 300 k, where p / 300 is still k - 1 for k > 0
        for p in _ulps(b, 3) + _ulps(300.0 * k, 3):
            if np.trunc(p * INV) != np.trunc(p / 300.0):
                disagree.append(p)
            vals.append(p)
    assert len(disagree) > 20, "the disagreement points were not reached"
    vals = np.unique(np.asarray(vals, np.float64))
    return vals, np.asarray(disagree, np.float64)


# ---------------------------------------------------------------- far from the world origin -------------------------------------------

@pytest.mark.parametrize("base", [(3.0e6 + 17.25, -2.0e5 + 0.5, -7.5e6 + 3.125), (3.9e7 + 0.75, -3.9e7 - 0.25, 3.9e7 + 150.5)], ids=["3e6", "3.9e7"])
def test_far_from_origin_device_frames(ctx, oracle, base):
    """A 100 k scene thousands of km out (the second one just inside the packed key's range on every axis), then frames of device adds,
    removes and sets with in-cell movers and changers, every batch on the device path."""
    rng = np.random.default_rng(61)
    base = np.asarray(base, np.float64)
    n = 100_000
    w = Edge(ctx, oracle, 160_000, _views_at(base))
    pos = base + (rng.random((n, 3)) * 2 - 1) * np.array([2500.0, 250.0, 2500.0])
    rad = (0.25 + 6 * rng.random(n)).astype(np.float32)
    rad[rng.random(n) < 0.01] = np.float32(320.0)
    assert (_cells(pos) >= KEY_LO).all() and (_cells(pos) <= KEY_HI).all()
    w.host_add(np.arange(n, dtype=np.int32), (np.arange(n) % 3).astype(np.uint8), pos, rad)
    next_id = n
    for frame in range(2):
        k = 6000
        p = base + (rng.random((k, 3)) * 2 - 1) * np.array([3000.0, 250.0, 3000.0])
        r = (0.5 + 4 * rng.random(k)).astype(np.float32)
        ids = np.arange(next_id, next_id + k, dtype=np.int32)
        next_id += k
        assert w.launches(w.add, ids, rng.integers(0, 4, k).astype(np.uint8), p, r, max_entity=next_id) >= 4
        w.check(f"frame {frame}: adds", mirror=False)
        live = np.nonzero(w.alive)[0]
        w.remove(rng.choice(live, 4000, replace=False).astype(np.int32))
        w.check(f"frame {frame}: removes", mirror=False)
        live = np.nonzero(w.alive)[0]
        mv = rng.choice(live, 30_000, replace=False).astype(np.int32)
        step = np.where(rng.random((len(mv), 1)) < 0.5, 0.01, 250.0)  # half stay in their cell (mostly), half change it (mostly)
        newr = w.rad[mv].copy()
        newr[:200] = np.float32(310.0)  # is_big flips
        got = w.launches(w.set, mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * step, newr, max_entity=next_id, what=f"frame {frame}")
        assert got >= 5, "the batch left the device path"
        w.check(f"frame {frame}: set", mirror=frame == 1)
        w.check_mask_and_stats(w.views[2], f"frame {frame}")
    w.close()


# ---------------------------------------------------------------- cell 0, negative cells, rounding borders ---------------------------

def test_cell_zero_negative_cells_and_rounding_borders(ctx, oracle):
    """Movers that cross 0 inside cell 0 are in-place, ones that cross +-300 change cell; entities on exact multiples of 300 (negative
    ones too) and a few ulps either side of the points where trunc(p * f64(f32(1/300))) and trunc(p / 300) disagree, up to cell +-1e5:
    device adds, sets among those points, removes."""
    rng = np.random.default_rng(7)
    vals, disagree = _border_positions(rng)
    views = _views_at((0.0, 0.0, 0.0), 1500.0) + _views_at((300.0 * 33_333, 0.0, -300.0 * 33_333), 2000.0) + \
        _views_at((-300.0 * 99_999, 0.0, 300.0 * 100_000), 2000.0) + _views_at((300.0 * 4096, -300.0 * 77, 300.0), 2000.0)
    w = Edge(ctx, oracle, 200_000, views)
    base_pos = (rng.random((20_000, 3)) * 2 - 1) * np.array([1500.0, 150.0, 1500.0])
    w.host_add(np.arange(20_000, dtype=np.int32), np.zeros(20_000, np.uint8), base_pos, np.full(20_000, 2.0, np.float32))
    # in-place movers across 0 inside cell 0: not changers
    zero = np.array([[-10.0, 5.0, -20.0], [-299.0, -299.0, 299.0], [10.0, -10.0, 0.0], [299.0, 0.5, -0.5]])
    ids0 = np.arange(30_000, 30_004, dtype=np.int32)
    w.add(ids0, np.zeros(4, np.uint8), zero, np.full(4, 3.0, np.float32), max_entity=199_999)
    assert w.set(ids0, -zero, np.full(4, 3.0, np.float32), max_entity=199_999, what="across 0 inside cell 0") == 0
    across = np.array([[299.0, 1.0, 1.0], [-299.0, 1.0, 1.0], [1.0, 299.5, -1.0], [1.0, -1.0, -299.5]])
    assert w.set(ids0, across, np.full(4, 3.0, np.float32), max_entity=199_999) == 0
    assert w.set(ids0, across + np.array([[2.0, 0, 0], [-2.0, 0, 0], [0, 1.0, 0], [0, 0, -1.0]]), np.full(4, 3.0, np.float32), max_entity=199_999) == 4
    w.check("cell 0 and +-300")
    # border entities: every value on one axis, the others from the same set or plain
    k = 3000
    ax = rng.integers(0, 3, k)
    pos = (rng.random((k, 3)) * 2 - 1) * 1200.0
    pos[np.arange(k), ax] = rng.choice(vals, k)
    pos[: len(disagree), 0] = disagree  # every disagreement point once on x, also on z for some
    pos[len(disagree): 2 * len(disagree), 2] = disagree
    ids = np.arange(40_000, 40_000 + k, dtype=np.int32)
    w.add(ids, rng.integers(0, 3, k).astype(np.uint8), pos, np.full(k, 1.5, np.float32), max_entity=199_999)
    w.check("border adds")
    # sets among the border values: to a neighbouring ulp (a cell change exactly where the two formulas disagree), to another border value
    for rnd in range(3):
        mv = ids[rng.random(k) < 0.6]
        newp = w.pos[mv].copy()
        a = rng.integers(0, 3, len(mv))
        cur = newp[np.arange(len(mv)), a]
        pick = rng.random(len(mv))
        newp[np.arange(len(mv)), a] = np.where(pick < 0.4, np.nextafter(cur, np.where(rng.random(len(mv)) < 0.5, -np.inf, np.inf)),
                                               np.where(pick < 0.8, rng.choice(vals, len(mv)), -cur))
        got = w.set(mv, newp, w.rad[mv], max_entity=199_999, what=f"border round {rnd}")
        assert got > 0
        w.check(f"border round {rnd}", mirror=rnd == 2)
    w.remove(ids[::3])
    w.check("border removes")
    w.check_mask_and_stats(views[2], "borders")
    w.close()


# ---------------------------------------------------------------- is_big threshold and bad radii -------------------------------------

def test_is_big_threshold_and_bad_radii(ctx, oracle):
    """Radii 300.0f and its float neighbours flip is_big both ways in one batch; negative and NaN radii arrive by set and by add and
    switch plane masking off; it is back on once they are gone."""
    rng = np.random.default_rng(13)
    w = Edge(ctx, oracle, 60_000, _views_at((0.0, 0.0, 0.0), 2500.0))
    n = 30_000
    pos = (rng.random((n, 3)) * 2 - 1) * np.array([2500.0, 250.0, 2500.0])
    t300 = np.float32(300.0)
    up, down = np.nextafter(t300, np.float32(np.inf)), np.nextafter(t300, np.float32(0))
    rad = rng.choice(np.array([1.0, t300, up, down, 450.0], np.float32), n)
    w.host_add(np.arange(n, dtype=np.int32), (np.arange(n) % 2).astype(np.uint8), pos, rad)
    w.check("threshold radii", mirror=False)
    assert w.cs.lastLaunch()["plane_masking"]
    for rnd in range(2):
        mv = rng.choice(n, 9000, replace=False).astype(np.int32)
        old = w.rad[mv]
        flip = np.where(old > 300.0, rng.choice(np.array([t300, down], np.float32), len(mv)), up)  # big -> not big, not big -> big
        flip[::5] = old[::5]  # some keep their radius
        got = w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * 0.5, flip, max_entity=n - 1, what=f"flip {rnd}")
        assert got > 1000
        w.check(f"flip {rnd}", mirror=rnd == 1)
    bad = np.array([-1.0, -0.0, -5.0, np.nan, -1e-30, -400.0], np.float32)
    nan_neg = np.array([0xFFC00000], np.uint32).view(np.float32)[0]
    mv = rng.choice(n, 600, replace=False).astype(np.int32)
    br = rng.choice(np.append(bad, nan_neg).astype(np.float32), len(mv))
    w.set(mv, w.pos[mv], br, max_entity=n - 1, what="bad radii by set")
    add_ids = np.arange(n, n + 300, dtype=np.int32)
    ar = rng.choice(np.append(bad, [1.0, 2.0]).astype(np.float32), 300)
    w.add(add_ids, np.zeros(300, np.uint8), (rng.random((300, 3)) * 2 - 1) * 800.0, ar, max_entity=59_999)
    w.check_culls("bad radii")
    assert not w.cs.lastLaunch()["plane_masking"]
    assert np.array_equal(_bits([w.cs.getRadius(int(e)) for e in mv[:30]]), _bits(w.rad[mv[:30]]))
    w.set(mv, w.pos[mv], np.full(len(mv), 2.0, np.float32), max_entity=n + 300, what="bad radii repaired")
    w.check_culls("set back")
    assert not w.cs.lastLaunch()["plane_masking"], "the added bad radii are still there"
    w.remove(add_ids[~(ar >= 0)])
    w.check_culls("bad radii removed")
    assert w.cs.lastLaunch()["plane_masking"]
    w.check_mirror()
    w.close()


# ---------------------------------------------------------------- the packed key's range ---------------------------------------------

def test_packed_key_range_extremes_stay_on_the_device(ctx, oracle):
    """Cells -131 072 and 131 071 on every axis: device adds into them and sets between and inside them run the device kernels and equal
    the oracle."""
    rng = np.random.default_rng(17)
    corners = [np.array(c) for c in ((KEY_LO, KEY_LO, KEY_LO), (KEY_HI, KEY_HI, KEY_HI), (KEY_LO, KEY_HI, 0), (KEY_HI, 0, KEY_LO))]
    views = []
    for c in corners[:2]:
        views += _views_at(c * 300.0 + np.where(c >= 0, 150.0, -150.0), 1500.0)
    w = Edge(ctx, oracle, 20_000, views)
    w.host_add(np.arange(1000, dtype=np.int32), np.zeros(1000, np.uint8), (rng.random((1000, 3)) * 2 - 1) * 1000.0, np.full(1000, 2.0, np.float32))
    ids = np.arange(1000, 1000 + 4 * 300, dtype=np.int32)
    pos = np.concatenate([_in_cell(rng, c, 300) for c in corners])
    rad = (1.0 + rng.random(len(ids))).astype(np.float32)
    rad[::50] = 350.0
    assert w.launches(w.add, ids, rng.integers(0, 3, len(ids)).astype(np.uint8), pos, rad, max_entity=19_999) >= 4, "the add left the device path"
    w.check_culls("adds at the key range's ends")
    # sets: in place inside the extreme cells, and from one extreme corner to the other
    mv = ids[::2]
    newp = w.pos[mv] + rng.normal(size=(len(mv), 3)) * 0.01
    newp[::3] = _in_cell(rng, corners[0], len(newp[::3]))
    newp[1::3] = _in_cell(rng, corners[1], len(newp[1::3]))
    assert w.launches(w.set, mv, newp, w.rad[mv], max_entity=19_999, what="between the extremes") >= 5, "the set left the device path"
    w.check("sets at the key range's ends")
    w.close()


def _alias_cells(axis):
    a = np.array([5, 2, -3])
    b = a.copy()
    b[axis] += ALIAS
    near = a.copy()
    near[axis] += 1
    return a, b, near


@pytest.mark.parametrize("axis", [0, 1, 2], ids=["x", "y", "z"])
@pytest.mark.parametrize("way", ["device_add", "host_adds_then_set", "set_into_alias"])
def test_chains_a_key_period_apart_stay_apart(ctx, oracle, axis, way):
    """Two chains whose cells differ by 262 144 on one axis, everything else equal, share their packed device key.  Reached by a device
    add into an empty system, by host adds followed by a set_many_device batch (device tables built from a mirror with both chains), and by
    a device set that moves entities from a near chain into the far alias of an existing chain.  Both chains keep their own cell, and a
    host add into the far one afterwards equals the oracle."""
    rng = np.random.default_rng(100 + axis)
    a, b, near = _alias_cells(axis)
    center = lambda c: c * 300.0 + np.where(c >= 0, 150.0, -150.0)  # noqa: E731
    w = Edge(ctx, oracle, 10_000, _views_at(center(a), 1200.0) + _views_at(center(b), 1200.0))
    pa, pb, pn = _in_cell(rng, a, 250), _in_cell(rng, b, 180), _in_cell(rng, near, 220)
    ra, rb, rn = (np.full(k, 2.0, np.float32) for k in (250, 180, 220))
    ia, ib, i_near = np.arange(0, 250), np.arange(1000, 1180), np.arange(2000, 2220)
    if way == "device_add":
        ids = np.concatenate([ia, ib]).astype(np.int32)
        perm = rng.permutation(len(ids))
        w.add(ids[perm], np.zeros(len(ids), np.uint8), np.concatenate([pa, pb])[perm], np.concatenate([ra, rb])[perm], max_entity=9_999)
        w.check("device add of both chains")
    elif way == "host_adds_then_set":
        w.host_add(ia.astype(np.int32), np.zeros(250, np.uint8), pa, ra)
        w.host_add(ib.astype(np.int32), np.zeros(180, np.uint8), pb, rb)
        w.host_add(i_near.astype(np.int32), np.zeros(220, np.uint8), pn, rn)
        # in-cell movers in both chains, changers from the near chain into both
        mv = np.concatenate([ia[:100], ib[:100], i_near[:120]]).astype(np.int32)
        newp = np.concatenate([pa[:100] + 0.01, pb[:100] - 0.01, _in_cell(rng, a, 60), _in_cell(rng, b, 60)])
        w.set(mv, newp, w.rad[mv], max_entity=9_999, what="host-built tables with both chains")
        w.check("set over a mirror with both chains")
    else:
        w.host_add(ia.astype(np.int32), np.zeros(250, np.uint8), pa, ra)
        w.host_add(i_near.astype(np.int32), np.zeros(220, np.uint8), pn, rn)
        w.set(i_near[:5].astype(np.int32), pn[:5] + 0.01, rn[:5], max_entity=9_999)  # in place: the device is authoritative
        mv = i_near[20:170].astype(np.int32)
        w.set(mv, _in_cell(rng, b, len(mv)), w.rad[mv], max_entity=9_999, what="near chain into the far alias")
        w.check("set into the alias of an existing chain")
    # the far chain takes host adds afterwards like the oracle's
    extra = np.arange(3000, 3050, dtype=np.int32)
    w.host_add(extra, np.zeros(50, np.uint8), _in_cell(rng, b, 50), np.full(50, 1.0, np.float32))
    w.check("host add into the far chain")
    # once no chain lies outside the key's range, batches run on the device again
    far = np.nonzero(w.alive & (np.abs(_cells(w.pos)).max(axis=1) > KEY_HI))[0].astype(np.int32)
    w.remove(far)
    w.check_culls("far chain removed")
    live = np.nonzero(w.alive)[0].astype(np.int32)
    assert w.launches(w.set, live, w.pos[live] + 0.001, w.rad[live], max_entity=9_999) >= 1, "in-range batches stay on the host"
    w.check("back on the device")
    w.close()


# ---------------------------------------------------------------- the type range -----------------------------------------------------

def _check_types(w, what):
    """Entity count, per-type counts / offsets / n_types of the cull result, culls filtered to every present type, cull_views with
    per-view filters, and a pinned and a pageable destination, against the oracle."""
    cs, oc = w.cs, w.oc
    assert cs.entity_count() == int(w.alive.sum()), what
    counts = np.bincount(w.type[w.alive], minlength=256)
    present = np.nonzero(counts)[0]
    f_all, f_persp = w.views[2], w.views[0]
    fb = lb.culling.frustum_bytes(f_all)
    oids, otys, _ = oc.cull(fb)
    res = cs.cull(f_all)
    assert res.total == len(oids) and np.array_equal(_canon(res), np.sort(oids.astype(np.int64) * 256 + otys)), what
    vis = np.bincount(otys, minlength=256)
    assert np.array_equal(res.type_count, vis), f"{what}: type counts"
    assert np.array_equal(res.type_offset, np.concatenate([[0], np.cumsum(vis)[:-1]])), f"{what}: type offsets"
    assert int(res.raw.n_types) == (int(present.max()) + 1 if len(present) else 0), f"{what}: n_types"
    fpb = lb.culling.frustum_bytes(f_persp)
    for t in present:
        r = cs.cull(f_persp, int(t))
        i2, t2, _ = oc.cull(fpb, type=int(t))
        assert r.total == len(i2) and np.array_equal(np.sort(r.ids.astype(np.int64)), np.sort(i2.astype(np.int64))), f"{what}: type {t}"
        assert set(np.unique(r.types()).tolist()) <= {int(t)}
    # several views, one filter each
    filters = [254, 0, 0xFF, 128]
    frusta = [f_persp, w.views[1], f_all, f_all]
    base = np.concatenate([[0], np.cumsum(counts)[:-1]])
    for v, (ptr, r) in enumerate(cs.cull_views(frusta, filters)):
        i2, t2, _ = oc.cull(lb.culling.frustum_bytes(frusta[v]), type=-1 if filters[v] == 0xFF else filters[v])
        assert r.total == len(i2), f"{what}: view {v}"
        assert np.array_equal(np.ctypeslib.as_array(r.type_offset), base), f"{what}: view {v} type offsets"
        got = []
        for t in np.nonzero(np.ctypeslib.as_array(r.type_count))[0]:
            got.append(ctx_ids(w.ctx, ptr + 4 * int(base[t]), int(r.type_count[t])).astype(np.int64) * 256 + int(t))
        got = np.sort(np.concatenate(got + [np.zeros(0, np.int64)]))
        assert np.array_equal(got, np.sort(i2.astype(np.int64) * 256 + t2)), f"{what}: view {v} filter {filters[v]}"
    # pinned (cull()) and pageable destinations
    pinned = cs.cull(f_all)
    pageable = np.zeros(max(cs.entity_count(), 1), np.uint32)
    raw = _lib.CullResult()
    rc = cs.L.lb200_culling_cull(cs.h, C.byref(f_all), C.c_uint8(0xFF), pageable.ctypes.data_as(C.c_void_p), C.c_uint32(len(pageable)), C.byref(raw))
    assert rc == 0 and raw.total == pinned.total == len(oids), what
    for t in present:
        o, c = int(raw.type_offset[t]), int(raw.type_count[t])
        exp = np.sort(oids[otys == t].astype(np.int64))
        assert np.array_equal(np.sort(pageable[o:o + c].astype(np.int64)), exp), f"{what}: pageable type {t}"
        assert np.array_equal(np.sort(pinned.of_type(int(t)).astype(np.int64)), exp), f"{what}: pinned type {t}"


def ctx_ids(ctx, ptr, n):
    return ctx.copy_to_host(ptr, n, np.uint32) if n else np.zeros(0, np.uint32)


@pytest.mark.parametrize("kind", ["sparse", "all"])
def test_type_range(ctx, oracle, kind):
    """Types {0, 1, 7, 31, 32, 128, 200, 253, 254} or all of 0-254 (one cell holds 255 chains that differ only in type) through device
    adds, removes and sets; removing every entity of type 254 brings its count back to zero."""
    rng = np.random.default_rng(23 if kind == "sparse" else 29)
    tset = np.array([0, 1, 7, 31, 32, 128, 200, 253, 254] if kind == "sparse" else np.arange(255), np.uint8)
    w = Edge(ctx, oracle, 40_000, _views_at((0.0, 0.0, 0.0), 2000.0))
    k = 12_000
    pos = (rng.random((k, 3)) * 2 - 1) * np.array([2000.0, 200.0, 2000.0])
    types = tset[np.arange(k) % len(tset)]
    crowd = np.arange(0, 3 * 255)  # the first entities: one cell, every type several times
    pos[crowd] = _in_cell(rng, (1, 0, -2), len(crowd))
    rad = (0.5 + 3 * rng.random(k)).astype(np.float32)
    rad[rng.random(k) < 0.02] = 330.0
    ids = rng.permutation(k).astype(np.int32)
    w.add(ids, types, pos, rad, max_entity=39_999)
    _check_types(w, "device add")
    w.remove(rng.choice(ids, 3000, replace=False).astype(np.int32))
    _check_types(w, "device remove")
    live = np.nonzero(w.alive)[0].astype(np.int32)
    mv = rng.choice(live, len(live) // 2, replace=False).astype(np.int32)
    w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * np.array([250.0, 5.0, 250.0]), w.rad[mv], max_entity=39_999, what="types")
    _check_types(w, "device set")
    more = np.arange(20_000, 20_000 + 2 * len(tset), dtype=np.int32)
    w.add(more, np.repeat(tset, 2), _in_cell(rng, (1, 0, -2), len(more)), np.full(len(more), 1.0, np.float32), max_entity=39_999)
    _check_types(w, "second add into the crowded cell")
    w.remove(np.nonzero(w.alive & (w.type == 254))[0].astype(np.int32))
    _check_types(w, "type 254 removed")
    res = w.cs.cull(w.views[2])
    assert res.type_count[254] == 0 and int(np.bincount(w.type[w.alive], minlength=256)[254]) == 0
    w.check_mirror()
    w.close()


def test_sort_keys_over_types_they_do_not_draw(ctx, oracle):
    """createSortKeys after device adds, removes and sets of a scene where types 1 and 4-254 sit among meshes and decals."""
    rng = np.random.default_rng(37)
    n = 6000
    scene = scenes.cull_scene(n, (1500.0, 200.0, 1500.0), seed=38, type_probs=(0.5, 0.1, 0.1, 0.1, 0.2))
    types = scene["types"].copy()
    other = types == 4
    types[other] = rng.integers(4, 255, int(other.sum())).astype(np.uint8)
    sk = scenes.sortkey_setup(n, types, scene["pos"], seed=39)
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    a = scenes.c1_frustum_args()
    w = Edge(ctx, oracle, n, [lb.frustum_perspective(**dict(a, far=1500.0))])
    half = np.arange(0, n, 2, dtype=np.int32)
    w.host_add(half, types[half], scene["pos"][half], scene["radius"][half])
    rest = np.arange(1, n, 2, dtype=np.int32)
    w.add(rest, types[rest], scene["pos"][rest], scene["radius"][rest], max_entity=n - 1)
    w.remove(rng.choice(n, 900, replace=False).astype(np.int32))
    live = np.nonzero(w.alive)[0].astype(np.int32)
    mv = rng.choice(live, 2000, replace=False).astype(np.int32)
    w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * 150.0, w.rad[mv], max_entity=n - 1, what="sort-key scene")
    f = w.views[0]
    view = sortkeys.make_view(a["position"], a["position"], 1.0 / 60.0, 1.0, 1, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
    w.cs.cull_device(f, want_counts=False)
    got = S.read(S.createSortKeys(w.cs, view))
    oids, otys, _ = w.oc.cull(lb.culling.frustum_bytes(f))
    assert len(np.unique(otys)) > 10
    exp = oracle.create_sort_keys(oids, otys, sk["transforms"], sk["model_of"], sk["lod"].copy(), sk["flags"], sk["pose_frame"].copy(), sk["decal_sort_key"],
                                  sk["decal_layer"], sk["models"], sk["meshes"], view)
    assert np.array_equal(got["keys"], exp["keys"])
    assert np.array_equal(got["group_count"], exp["group_count"])
    S.close()
    w.close()


# ---------------------------------------------------------------- batch size: the tiled changer sort ---------------------------------

def test_changer_sort_on_its_tiled_path(ctx, oracle):
    """One set_many_device batch of 2.5 M entities, every one shifted 600 m in x: 2.5 M changers, above 2 x SMs x 8192 whatever the
    co-resident sort grid, so the changer sort takes its tiled path; plan and place behind it must still equal the oracle."""
    n = 2_500_000
    scene = scenes.cull_scene(n, (6000.0, 300.0, 6000.0), seed=71, big_fraction=0.002, type_probs=(0.7, 0.2, 0.1))
    w = Edge(ctx, oracle, n, _views_at((600.0, 0.0, 0.0), 3500.0))
    w.host_add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    ids = scene["entities"]
    got = w.set(ids, w.pos[ids] + np.array([600.0, 0.0, 0.0]), w.rad[ids], max_entity=n - 1, what="every entity shifted 600 m")
    assert got == n
    w.check("tiled changer sort")
    w.close()


# ---------------------------------------------------------------- freed pages, mask rows, statistics --------------------------------

def test_freed_pages_reused_within_one_batch(ctx, oracle):
    """In one batch a chain empties out (its open page and its full pages), another chain loses only its open page while its full pages
    stay, and the batch's changers open new pages: they take the freed ones, so no page id reaches the page count from before.  Mask rows
    and page statistics of culls after the batch hold, a page freed by the batch and reused later has a zero mask row, and a host add
    into the emptied chain equals the oracle."""
    rng = np.random.default_rng(43)
    w = Edge(ctx, oracle, 20_000, _views_at((0.0, 0.0, 0.0), 6500.0))
    # chains of 450 (pages 200 + 200 + 50: the open page holds 50) and 420 entities in cells of their own, and background
    pa, pb = _in_cell(rng, (12, 0, -13), 450), _in_cell(rng, (-14, 0, -11), 420)
    bg = (rng.random((5000, 3)) * 2 - 1) * np.array([2500.0, 200.0, 2500.0])
    ia, ib, ibg = np.arange(450, dtype=np.int32), np.arange(1000, 1420, dtype=np.int32), np.arange(2000, 7000, dtype=np.int32)
    w.host_add(ia, np.zeros(450, np.uint8), pa, np.full(450, 1.0, np.float32))
    w.host_add(ib, np.zeros(420, np.uint8), pb, np.full(420, 1.0, np.float32))
    w.host_add(ibg, np.zeros(5000, np.uint8), bg, np.full(5000, 1.0, np.float32))
    pages = w.cs.pages()
    n_pages = len(pages)
    assert int(w.cs.page_ids().max()) == n_pages - 1, "a freshly uploaded scene has no free pages"
    open_a = [p for p in pages if tuple(p["indices"]) == (12, 0, -13) and p["count"] == 50][0]["entities"]
    w.check_culls("before")
    # one batch: chain b empties (3 pages), chain a loses its open page (1); its 470 changers open 4 pages in two new cells
    mv = np.concatenate([ib, open_a]).astype(np.int32)
    newp = np.concatenate([_in_cell(rng, (16, 0, 15), 240), _in_cell(rng, (-17, 0, 14), 230)])
    assert w.set(mv, newp, w.rad[mv], max_entity=19_999, what="pages freed and reused") == len(mv)
    w.check_culls("after the batch")
    w.check_mask_and_stats(w.views[2], "after the batch")
    ids_after = w.cs.page_ids()
    assert ids_after.max() < n_pages, f"page ids {ids_after.max()} >= {n_pages}: the batch did not reuse its freed pages"
    w.check_mirror()
    # a device remove frees pages again; a cull, then a host add into a new cell reuses one of them: its row is zero
    w.remove(ia[:200])
    w.check_mask_and_stats(w.views[2], "after a device remove")
    before = set(w.cs.page_ids().tolist())
    w.host_add(np.array([9000], np.int32), np.zeros(1, np.uint8), _in_cell(rng, (19, 0, 19), 1), np.array([1.0], np.float32))
    ids_now = w.cs.page_ids()
    new = [i for i, p in enumerate(ids_now.tolist()) if p not in before]
    assert len(new) == 1 and ids_now[new[0]] < n_pages, "the new cell did not take a freed page"
    assert not w.cs.read_bitmask()[new[0]].any(), "a freed page kept a mask row"
    # host adds into the emptied chain
    w.host_add(np.arange(9100, 9130, dtype=np.int32), np.zeros(30, np.uint8), _in_cell(rng, (-14, 0, -11), 30), np.full(30, 1.0, np.float32))
    w.check("host add into the emptied chain")
    w.close()
