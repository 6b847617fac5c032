"""Device adds and removes (CullingSystem.add_many_device / remove_many_device, csrc/culling_rebin.cu) against the oracle's sequential
CullingSystem::add / remove / set: the same visible sets over several views (perspective and ortho) after every batch, and a host mirror
that, pulled back from the device, holds every live entity in the cell of its position with its exact sphere."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys

gpu = pytest.mark.gpu


def _canon(res):
    return np.sort(res.ids.astype(np.int64) * 256 + res.types())


def _views(far=3000.0, ortho=5000.0):
    a = scenes.c1_frustum_args()
    return [lb.frustum_perspective(**dict(a, far=far)),
            lb.frustum_perspective(**dict(a, position=(700.0, 20.0, -400.0), direction=(-0.7, -0.05, 0.7), far=far - 500.0)),
            lb.frustum_ortho((0.0, 0.0, ortho), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), ortho, ortho, 0.0, 2 * ortho)]


def _bits(r):
    return np.asarray(r, np.float32).view(np.uint32)


class Twin:
    """A CullingSystem edited on the device next to the oracle edited sequentially, and the sphere / type / liveness every id should have."""

    def __init__(self, ctx, oracle, cap, views):
        self.ctx, self.cs, self.oc, self.views = ctx, lb.CullingSystem(ctx), oracle.OracleCulling(), views
        self.pos = np.zeros((cap, 3), np.float64)
        self.rad = np.zeros(cap, np.float32)
        self.type = np.zeros(cap, np.uint8)
        self.alive = np.zeros(cap, bool)

    def _dev(self, *arrays):
        return [self.ctx.to_device(np.ascontiguousarray(a)) for a in arrays]

    def _free(self, ptrs):
        for p in ptrs:
            self.ctx.free_device(p)

    def host_add(self, ids, types, pos, rad):
        self.cs.add(ids, types, pos, rad)
        self.oc.add(ids, types, pos, rad)
        self._added(ids, types, pos, rad)

    def _added(self, ids, types, pos, rad):
        self.pos[ids], self.rad[ids], self.type[ids], self.alive[ids] = pos, rad, types, True

    def add(self, ids, types, pos, rad, max_entity, identity=False):
        ids = np.asarray(ids, np.int32)
        types, rad = np.asarray(types, np.uint8), np.asarray(rad, np.float32)
        d = self._dev(ids, types, pos, rad)
        self.cs.add_many_device(d[2], d[3], d[1], len(ids), dev_entities=None if identity else d[0], max_entity=max_entity)
        self._free(d)
        self.oc.add(ids, types, pos, rad)
        self._added(ids, types, pos, rad)

    def remove(self, ids):
        ids = np.asarray(ids, np.int32)
        d = self._dev(ids)
        self.cs.remove_many_device(d[0], len(ids))
        self._free(d)
        self.oc.remove(ids)
        ok = (ids >= 0) & (ids < len(self.alive))
        self.alive[ids[ok]] = False

    def set(self, ids, pos, rad, max_entity):
        ids = np.asarray(ids, np.int32)
        d = self._dev(ids, pos, rad)
        self.cs.set_many_device(d[1], d[2], len(ids), dev_entities=d[0], max_entity=max_entity)
        self._free(d)
        self.oc.set(ids, pos, rad)
        self.pos[ids], self.rad[ids] = pos, rad

    def check_culls(self, what):
        out = []
        for k, f in enumerate(self.views):
            res = self.cs.cull(f)
            oi, ot, _ = self.oc.cull(lb.culling.frustum_bytes(f))
            assert res.total == len(oi) and np.array_equal(_canon(res), np.sort(oi.astype(np.int64) * 256 + ot)), f"{what}: view {k}"
            out.append(_canon(res))
        return out

    def check_counters(self, sample, radius_first=False):
        """entity_count, get_radius and is_added answer for the device state without a sync_host first.  entity_count never pulls the
        device state back; of the other two, the one called first (radius_first) does."""
        assert self.cs.entity_count() == int(self.alive.sum())
        live = sample[self.alive[sample]]

        def radii():
            assert np.array_equal(_bits([self.cs.getRadius(int(e)) for e in live[:40]]), _bits(self.rad[live[:40]]))

        if radius_first:
            radii()
        assert [self.cs.isAdded(int(e)) for e in sample] == [bool(self.alive[e]) for e in sample]
        if not radius_first:
            radii()

    def check_mirror(self):
        self.cs.sync_host()
        seen = np.zeros(len(self.alive), bool)
        for pg in self.cs.pages():
            e = pg["entities"]
            assert pg["count"] == len(e) and 0 < len(e) <= 200 and not seen[e].any()
            seen[e] = True
            key = (self.pos[e] * np.float32(1 / 300.0)).astype(np.int64)  # trunc toward zero like IVec3(DVec3)
            assert np.all(key == np.asarray(pg["indices"])[None, :]) and np.all((self.rad[e] > 300.0) == bool(pg["is_big"]))
            assert np.all(self.type[e] == pg["type"])
            assert np.array_equal(pg["spheres"][:, :3], (self.pos[e] - np.asarray(pg["origin"])).astype(np.float32))
            assert np.array_equal(_bits(pg["spheres"][:, 3]), _bits(self.rad[e]))
        assert np.array_equal(seen, self.alive)
        assert self.cs.entity_count() == int(self.alive.sum())

    def close(self):
        self.cs.close()


def _spheres(rng, k, center, spread, big=0.02):
    pos = np.asarray(center, np.float64) + (rng.random((k, 3)) * 2.0 - 1.0) * np.asarray(spread, np.float64)
    rad = (0.5 + 4.5 * rng.random(k)).astype(np.float32)
    b = rng.random(k) < big
    rad[b] = (300.0 + 350.0 * rng.random(int(b.sum()))).astype(np.float32)
    return pos, rad


def _cell_grid(k, origin, nx, ny):
    """k positions, one per 300 m cell of a grid nx x ny x (k / nx / ny) cells from `origin`: every one starts a chain."""
    i = np.arange(k)
    c = np.stack([i % nx, (i // nx) % ny, i // (nx * ny)], axis=1).astype(np.float64)
    return np.asarray(origin, np.float64) + c * 300.0 + 150.0


@gpu
def test_mixed_device_edits_equal_sequential_edits(ctx, oracle):
    """Frames of device adds (new ids above the range, into open pages and new cells, a 4,000-entity crowd into one cell, big radii),
    device removes (with ids never added and ids listed twice) and a set_many_device batch, culled after every frame."""
    rng = np.random.default_rng(31)
    n = 150_000
    scene = scenes.cull_scene(n, (3000.0, 300.0, 3000.0), seed=5, big_fraction=0.01, type_probs=(0.7, 0.2, 0.1))
    w = Twin(ctx, oracle, 400_000, _views())
    w.host_add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    next_id = n
    for frame in range(4):
        # adds: inside the scene (open pages of existing chains, type 3 starts new chains there), in new cells outside it, one crowd
        p_in, r_in = _spheres(rng, 3000, (0.0, 0.0, 0.0), (3000.0, 300.0, 3000.0))
        p_out, r_out = _spheres(rng, 1000, (4500.0 + 1000.0 * frame, 0.0, -1000.0), (1200.0, 300.0, 1200.0))
        p_crowd, r_crowd = _spheres(rng, 4000, (1234.0 + 300.0 * frame, 10.0, -777.0), (20.0, 5.0, 20.0), big=0.0)
        pos = np.concatenate([p_in, p_out, p_crowd])
        rad = np.concatenate([r_in, r_out, r_crowd])
        k = len(pos)
        ids = (next_id + rng.permutation(k)).astype(np.int32)
        types = rng.choice(np.array([0, 1, 2, 3], np.uint8), k, p=[0.6, 0.2, 0.1, 0.1]).astype(np.uint8)
        types[-len(p_crowd):] = 0  # the crowd: one chain
        next_id += k
        w.add(ids, types, pos, rad, max_entity=next_id + 1000)
        w.check_counters(np.concatenate([ids[:60], rng.choice(n, 60, replace=False).astype(np.int32)]))
        w.check_culls(f"frame {frame}: adds")
        # removes: live ids old and new, ids never added, ids removed before, ids listed twice
        live = np.nonzero(w.alive)[0]
        gone = rng.choice(live, 5000, replace=False).astype(np.int32)
        never = np.array([next_id + 5, next_id + 17, 399_999, -1, -100], np.int32)
        batch = np.concatenate([gone, gone[:300], never, gone[-50:]])
        w.remove(rng.permutation(batch).astype(np.int32))
        w.check_counters(np.concatenate([gone[:60], ids[:60]]), radius_first=True)
        w.check_culls(f"frame {frame}: removes")
        # a re-binning batch of live entities, old and new
        live = np.nonzero(w.alive)[0]
        mv = rng.choice(live, 20_000, replace=False).astype(np.int32)
        w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * np.array([200.0, 10.0, 200.0]), w.rad[mv], max_entity=next_id)
        w.check_culls(f"frame {frame}: set")
        if frame in (1, 3):
            w.check_mirror()
    w.close()


@gpu
def test_system_edited_only_on_the_device(ctx, oracle):
    """A system that starts empty and is only ever edited on the device (the identity id list too)."""
    rng = np.random.default_rng(5)
    w = Twin(ctx, oracle, 100_000, _views())
    assert w.cs.cull(w.views[0]).total == 0
    pos, rad = _spheres(rng, 20_000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    types = rng.choice(np.array([0, 1, 2], np.uint8), 20_000).astype(np.uint8)
    w.add(np.arange(20_000, dtype=np.int32), types, pos, rad, max_entity=19_999, identity=True)
    w.check_counters(rng.choice(20_000, 50, replace=False).astype(np.int32))
    w.check_culls("identity add into an empty system")
    w.remove(rng.choice(20_000, 10_000, replace=False).astype(np.int32))
    w.check_culls("half removed")
    pos, rad = _spheres(rng, 30_000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.add(np.arange(20_000, 50_000, dtype=np.int32), rng.choice(np.array([0, 1, 2], np.uint8), 30_000).astype(np.uint8), pos, rad, max_entity=60_000)
    w.check_culls("second add")
    w.check_mirror()
    w.close()


@gpu
def test_page_and_chain_edges(ctx, oracle):
    """Adds of 199, 200, 201 and 401 entities into empty cells (one page short, full, one over, two pages and one), a chain emptied whose
    open page heads it in the hash map and then refilled, a remove and re-add of the same ids in consecutive batches, and a system
    emptied by removes (the cull returns nothing)."""
    rng = np.random.default_rng(9)
    w = Twin(ctx, oracle, 20_000, _views())
    base_pos, base_rad = _spheres(rng, 2000, (0.0, 0.0, 0.0), (2000.0, 200.0, 2000.0))
    w.host_add(np.arange(2000, dtype=np.int32), np.zeros(2000, np.uint8), base_pos, base_rad)
    next_id = 2000
    cells = {}
    for j, k in enumerate((199, 200, 201, 401)):
        center = (-4350.0 + 300.0 * j, 150.0, -1050.0)  # empty cells (-14 + j, 0, -3), one per size, outside the base scene
        pos, rad = _spheres(rng, k, center, (140.0, 140.0, 140.0), big=0.0)
        ids = np.arange(next_id, next_id + k, dtype=np.int32)
        next_id += k
        w.add(ids, np.zeros(k, np.uint8), pos, rad, max_entity=next_id - 1)
        w.check_culls(f"{k} into an empty cell")
        cells[k] = ids
    w.cs.sync_host()
    per_cell = {}
    for pg in w.cs.pages():
        per_cell.setdefault(tuple(pg["indices"]), []).append(pg["count"])
    for j, k in enumerate((199, 200, 201, 401)):
        counts = per_cell[(-14 + j, 0, -3)]
        assert sum(counts) == k and len(counts) == (k + 199) // 200
    # empty the 401-entity chain (its open page is the one the hash map names), then add into the cell again
    w.set(cells[200][:10], w.pos[cells[200][:10]], w.rad[cells[200][:10]], max_entity=next_id)  # in place: the device is authoritative again
    w.remove(cells[401])
    w.check_culls("chain emptied")
    pos, rad = _spheres(rng, 250, (-3450.0, 150.0, -1050.0), (140.0, 140.0, 140.0), big=0.0)
    refill = np.arange(next_id, next_id + 250, dtype=np.int32)
    next_id += 250
    w.add(refill, np.zeros(250, np.uint8), pos, rad, max_entity=next_id)
    w.check_culls("chain refilled")
    # removed in one batch, added back (other spheres) in the next
    back = cells[201]
    w.remove(back)
    w.check_culls("removed")
    pos, rad = _spheres(rng, len(back), (0.0, 0.0, 0.0), (2000.0, 200.0, 2000.0))
    w.add(back, np.ones(len(back), np.uint8), pos, rad, max_entity=next_id)
    w.check_counters(back[:30], radius_first=True)
    w.check_culls("re-added")
    w.check_mirror()
    # every entity removed: nothing is visible, and adds work again afterwards
    w.remove(np.nonzero(w.alive)[0].astype(np.int32))
    assert w.cs.entity_count() == 0
    for f in w.views:
        assert w.cs.cull(f).total == 0
    w.check_culls("all removed")
    w.add(np.array([7], np.int32), np.array([2], np.uint8), np.array([[0.0, 0.0, -10.0]]), np.array([1.0], np.float32), max_entity=next_id)
    w.check_culls("one after all removed")
    w.check_mirror()
    w.close()


@gpu
def test_refused_batches_change_nothing(ctx, oracle):
    """A batch with an id added already, an id listed twice, an id above max_entity, a negative id or type 0xff returns
    LB200_ERR_INVALID; culls and the pulled-back pages equal those from before, and the new ids of the batch can be added afterwards."""
    rng = np.random.default_rng(12)
    w = Twin(ctx, oracle, 40_000, _views())
    pos, rad = _spheres(rng, 20_000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.host_add(np.arange(20_000, dtype=np.int32), rng.choice(np.array([0, 1], np.uint8), 20_000).astype(np.uint8), pos, rad)
    pos, rad = _spheres(rng, 3000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.add(np.arange(20_000, 23_000, dtype=np.int32), np.zeros(3000, np.uint8), pos, rad, max_entity=30_000)

    def pages():
        w.cs.sync_host()
        order = np.argsort(w.cs.page_ids())
        pg = w.cs.pages()
        return [(pg[i]["indices"], pg[i]["type"], pg[i]["is_big"], pg[i]["spheres"].tobytes(), pg[i]["entities"].tobytes()) for i in order]

    new = np.arange(25_000, 25_100, dtype=np.int32)
    cases = {"added already": (np.concatenate([new, [20_500]]), 0), "listed twice": (np.concatenate([new, new[5:6]]), 0),
             "above max_entity": (np.concatenate([new, [30_001]]), 0), "negative": (np.concatenate([new, [-3]]), 0),
             "type 0xff": (new, 0xff)}
    for what, (ids, bad_type) in cases.items():
        before_pages = pages()
        w.set(np.array([20_000], np.int32), w.pos[[20_000]], w.rad[[20_000]], max_entity=30_000)  # in place: the device is authoritative again
        before = w.check_culls(f"{what}: before")
        ids = ids.astype(np.int32)
        types = np.zeros(len(ids), np.uint8)
        types[-1] = bad_type
        p, r = _spheres(rng, len(ids), (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
        d = [ctx.to_device(a) for a in (ids, types, p, r)]
        with pytest.raises(lb.LumixB200Error) as err:
            w.cs.add_many_device(d[2], d[3], d[1], len(ids), dev_entities=d[0], max_entity=30_000)
        for x in d:
            ctx.free_device(x)
        assert err.value.code == _lib.ERR_INVALID, what
        assert w.cs.entity_count() == int(w.alive.sum())
        after = w.check_culls(f"{what}: after")
        assert all(np.array_equal(a, b) for a, b in zip(before, after)), what
        assert pages() == before_pages, what
        assert not any(w.cs.isAdded(int(e)) for e in new[:10])
    # the claims were released: the same new ids are accepted now
    p, r = _spheres(rng, len(new), (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.add(new, np.full(len(new), 2, np.uint8), p, r, max_entity=30_000)
    w.check_culls("accepted after the refusals")
    w.check_mirror()
    w.close()


@gpu
def test_growth_while_device_authoritative(ctx, oracle):
    """The entity -> slot table grows with its contents while the device is authoritative (adds with max_entity several times its size,
    set_many_device with a larger max_entity after an earlier batch), the chain hash map is rehashed at least twice (two batches of
    10,000 entities in 10,000 new cells each), and the page arrays and output ids grow."""
    rng = np.random.default_rng(44)
    n = 20_000
    views = _views() + [lb.frustum_ortho((0.0, 0.0, 40000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 40000.0, 40000.0, 0.0, 80000.0)]
    w = Twin(ctx, oracle, 2_000_000, views)
    pos, rad = _spheres(rng, n, (0.0, 0.0, 0.0), (3000.0, 300.0, 3000.0))
    w.host_add(np.arange(n, dtype=np.int32), rng.choice(np.array([0, 1, 2], np.uint8), n).astype(np.uint8), pos, rad)
    mv = rng.choice(n, 2000, replace=False).astype(np.int32)
    w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * 300.0, w.rad[mv], max_entity=n - 1)  # the entity -> slot table: 32 k entries
    w.check_culls("first batch")
    mv = rng.choice(n, 2000, replace=False).astype(np.int32)
    w.set(mv, w.pos[mv] + rng.normal(size=(len(mv), 3)) * 300.0, w.rad[mv], max_entity=300_000)  # grows while authoritative
    w.check_culls("set_many_device with a larger max_entity")
    # ids far above the table: 1.2 M entries needed
    ids = rng.choice(np.arange(600_000, 1_200_000), 5000, replace=False).astype(np.int32)
    pos, rad = _spheres(rng, 5000, (0.0, 0.0, 0.0), (3000.0, 300.0, 3000.0))
    w.add(ids, np.zeros(5000, np.uint8), pos, rad, max_entity=1_199_999)
    w.check_counters(np.concatenate([ids[:50], mv[:20]]))
    w.check_culls("adds far above the entity table")
    # new chains: every entity of a batch in its own cell, 10,000 cells per batch
    for b in range(3):
        k = 10_000
        pos = _cell_grid(k, (3300.0 + 12_000.0 * b, 0.0, 3300.0), 40, 20)
        pos += (rng.random(pos.shape) - 0.5) * 100.0
        rad = (1.0 + rng.random(k)).astype(np.float32)
        ids = np.arange(1_200_000 + b * k, 1_200_000 + (b + 1) * k, dtype=np.int32)
        w.add(ids, rng.choice(np.array([0, 3], np.uint8), k).astype(np.uint8), pos, rad, max_entity=1_999_999)
        res = w.check_culls(f"new cells, batch {b}")
        assert len(res[-1]) > 0.9 * w.alive.sum(), "the ortho view sees (nearly) everything"
    w.remove(np.arange(1_200_000, 1_205_000, dtype=np.int32))
    w.check_culls("removes after the growth")
    w.check_mirror()
    w.close()


@gpu
def test_bad_radii_switch_plane_masking(ctx, oracle):
    """Negative and +-NaN radii added on the device switch the cull's plane masking off (the culls still equal the oracle's); removing
    them switches it back on."""
    rng = np.random.default_rng(3)
    w = Twin(ctx, oracle, 40_000, _views())
    pos, rad = _spheres(rng, 30_000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.host_add(np.arange(30_000, dtype=np.int32), np.zeros(30_000, np.uint8), pos, rad)
    w.check_culls("clean")
    assert w.cs.lastLaunch()["plane_masking"]
    bad = np.array([-1.0, -0.0, -5.0, np.nan, np.nan, -1e-30, -400.0], np.float32)
    bad[4] = np.array([0xFFC00000], np.uint32).view(np.float32)[0]  # -NaN
    k = 700
    rad = np.concatenate([np.repeat(bad, k // len(bad)), (1.0 + rng.random(k - k // len(bad) * len(bad))).astype(np.float32)])
    pos, _ = _spheres(rng, k, (0.0, 0.0, -800.0), (800.0, 100.0, 800.0))
    ids = np.arange(30_000, 30_000 + k, dtype=np.int32)
    w.add(ids, np.zeros(k, np.uint8), pos, rad, max_entity=39_999)
    w.check_culls("bad radii added")
    has_bad = bool(np.any(~(rad >= 0)))
    assert w.cs.lastLaunch()["plane_masking"] == (not has_bad)
    w.check_counters(ids[::10], radius_first=True)
    w.remove(ids[~(rad >= 0)])
    w.check_culls("bad radii removed")
    assert w.cs.lastLaunch()["plane_masking"]
    w.check_mirror()
    w.close()


@gpu
def test_host_edits_between_device_edits(ctx, oracle):
    """A device add, then a host add (which pulls the device state back), then a device remove, then a cull."""
    rng = np.random.default_rng(17)
    w = Twin(ctx, oracle, 50_000, _views())
    pos, rad = _spheres(rng, 20_000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.host_add(np.arange(20_000, dtype=np.int32), np.zeros(20_000, np.uint8), pos, rad)
    pos, rad = _spheres(rng, 5000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.add(np.arange(20_000, 25_000, dtype=np.int32), np.ones(5000, np.uint8), pos, rad, max_entity=30_000)
    pos, rad = _spheres(rng, 5000, (0.0, 0.0, 0.0), (2500.0, 300.0, 2500.0))
    w.host_add(np.arange(30_000, 35_000, dtype=np.int32), np.full(5000, 2, np.uint8), pos, rad)
    gone = np.concatenate([rng.choice(20_000, 2000, replace=False), rng.choice(np.arange(20_000, 25_000), 2000, replace=False),
                           rng.choice(np.arange(30_000, 35_000), 2000, replace=False)]).astype(np.int32)
    w.remove(gone)
    w.check_culls("device add, host add, device remove")
    w.check_counters(gone[::100])
    w.check_mirror()
    w.close()


@gpu
def test_sort_keys_refuse_ids_a_device_add_put_beyond_max_entities(ctx, oracle):
    """createSortKeys indexes its entity records by the culled ids: after a device add of an id >= its max_entities it refuses; device
    removes and re-adds below max_entities keep it equal to the oracle."""
    n = 5000
    scene = scenes.cull_scene(n, (1500.0, 200.0, 1500.0), seed=8, type_probs=(0.85, 0.05, 0.05, 0.05))
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=9)
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    w = Twin(ctx, oracle, n + 10, [lb.frustum_perspective(**dict(scenes.c1_frustum_args(), far=1500.0))])
    w.host_add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    a = scenes.c1_frustum_args()
    f = w.views[0]

    def keys(frame):
        view = sortkeys.make_view(a["position"], a["position"], 1.0 / 60.0, 1.0, frame, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
        w.cs.cull_device(f, want_counts=False)
        got = S.read(S.createSortKeys(w.cs, view))
        oids, otys, _ = w.oc.cull(lb.culling.frustum_bytes(f))
        exp = oracle.create_sort_keys(oids, otys, sk["transforms"], sk["model_of"], sk["lod"].copy(), sk["flags"], sk["pose_frame"].copy(), sk["decal_sort_key"],
                                      sk["decal_layer"], sk["models"], sk["meshes"], view)
        assert np.array_equal(got["keys"], exp["keys"])

    gone = np.arange(0, n, 7, dtype=np.int32)
    w.remove(gone)
    w.add(gone, w.type[gone], w.pos[gone], w.rad[gone], max_entity=n - 1)
    keys(1)
    w.add(np.array([n], np.int32), np.zeros(1, np.uint8), np.array([[0.0, 0.0, -20.0]]), np.array([1.0], np.float32), max_entity=n)
    w.cs.cull_device(f, want_counts=False)
    view = sortkeys.make_view(a["position"], a["position"], 1.0 / 60.0, 1.0, 2, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
    launches = ctx.launches
    with pytest.raises(lb.LumixB200Error) as err:
        S.createSortKeys(w.cs, view)
    assert err.value.code == _lib.ERR_INVALID and ctx.launches == launches
    S.close()
    w.close()


def test_device_edits_without_a_device_change_nothing():
    """On a culling system without a context both device calls report NoDeviceError and leave the host state as it was."""
    cs = lb.CullingSystem(None)
    cs.add([1, 2, 300], [0, 1, 0], [(0.0, 0.0, -5.0), (10.0, 0.0, -5.0), (700.0, 0.0, 0.0)], [1.0, 2.0, 3.0])
    before = (cs.entity_count(), cs.page_count(), [(p["indices"], p["count"], p["entities"].tolist()) for p in cs.pages()])
    with pytest.raises(lb.NoDeviceError):
        cs.add_many_device(0x1000, 0x2000, 0x3000, 4, dev_entities=0x4000, max_entity=500)
    with pytest.raises(lb.NoDeviceError):
        cs.remove_many_device(0x4000, 2)
    assert (cs.entity_count(), cs.page_count(), [(p["indices"], p["count"], p["entities"].tolist()) for p in cs.pages()]) == before
    assert cs.isAdded(300) and not cs.isAdded(4) and cs.getRadius(2) == 2.0
    cs.close()
