"""GPU parity of CullingSystem::cull against the oracle (bit-exact visible sets per renderable type)."""
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes

pytestmark = pytest.mark.gpu


def _both(ctx, oracle, scene):
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    return cs, oc


def _assert_same(res, oids, otys):
    assert res.total == len(oids)
    got = np.sort(res.ids.astype(np.int64) * 256 + res.types())
    exp = np.sort(oids.astype(np.int64) * 256 + otys)
    assert np.array_equal(got, exp)


def _frustums():
    a = scenes.c1_frustum_args()
    yield "c1", a
    b = dict(a); b["position"] = (123.456, -20.0, 987.0); b["direction"] = (0.3, -0.1, -0.9); b["far"] = 900.0
    yield "tilted", b
    c = dict(a); c["position"] = (-1500.0, 50.0, -1500.0); c["direction"] = (1.0, 0.0, 1.0); c["far"] = 5000.0
    yield "diag_far", c
    d = dict(a); d["position"] = (1e6 + 0.25, 0.0, -2e6 + 0.5); d["far"] = 100.0
    yield "nothing", d


@pytest.mark.parametrize("name,args", list(_frustums()))
def test_c1_100k_matches_oracle(ctx, oracle, name, args):
    scene = scenes.c1_scene(100_000)
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_perspective(**args)
    fo = oracle.frustum_perspective(args["position"], args["direction"], args["up"], args["fov"], args["ratio"], args["near"], args["far"])
    assert bytes(f) == fo.tobytes()
    res = cs.cull(f)
    oids, otys, st = oc.cull(fo)
    _assert_same(res, oids, otys)
    assert res.stats["pages_tested"] == st["pages_tested"]
    assert res.stats["pages_inside"] == st["pages_inside"]
    assert res.stats["pages_outside"] == st["pages_outside"]
    assert res.stats["entities_tested"] == st["entities_tested"]


def test_types_big_and_filter(ctx, oracle):
    scene = scenes.cull_scene(300_000, (3000.0, 300.0, 3000.0), seed=11, big_fraction=0.01, type_probs=(0.6, 0.2, 0.1, 0.1))
    cs, oc = _both(ctx, oracle, scene)
    args = scenes.c1_frustum_args(); args["far"] = 2500.0
    f = lb.frustum_perspective(**args)
    fo = lb.culling.frustum_bytes(f)
    res = cs.cull(f)
    oids, otys, _ = oc.cull(fo)
    _assert_same(res, oids, otys)
    for t in range(5):
        r = cs.cull(f, t)
        i2, t2, _ = oc.cull(fo, type=t)
        _assert_same(r, i2, t2)
        assert set(np.unique(r.types())) <= {t}


def test_ortho_frustum(ctx, oracle):
    scene = scenes.c1_scene(50_000, seed=5)
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_ortho((10.0, 500.0, -20.0), (0.0, 1.0, 0.05), (0.0, 0.0, 1.0), 700.0, 400.0, 0.0, 1200.0)
    res = cs.cull(f)
    oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
    _assert_same(res, oids, otys)


def test_incremental_updates_and_bitmask(ctx, oracle):
    rng = np.random.default_rng(3)
    scene = scenes.c1_scene(60_000, seed=9)
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_perspective(**scenes.c1_frustum_args())
    fo = lb.culling.frustum_bytes(f)
    for step in range(4):
        n = 3000
        ids = rng.choice(60_000, n, replace=False).astype(np.int32)
        alive = np.array([cs.isAdded(int(i)) for i in ids])
        ids = ids[alive]
        third = len(ids) // 3
        mv, rs, rm = ids[:third], ids[third:2 * third], ids[2 * third:]
        newpos = scene["pos"][mv] + rng.normal(size=(len(mv), 3)) * np.array([400.0, 40.0, 400.0])
        cs.setPosition(mv, newpos); oc.set_position(mv, newpos)
        newrad = (rng.random(len(rs)) * 700.0).astype(np.float32)  # crosses the is_big threshold both ways
        cs.setRadius(rs, newrad); oc.set_radius(rs, newrad)
        cs.remove(rm); oc.remove(rm)
        res = cs.cull(f)
        oids, otys, _ = oc.cull(fo)
        _assert_same(res, oids, otys)
    # visibility bitmask (page, slot) agrees with the id list
    res = cs.cull(f)
    mask = cs.read_bitmask()
    pages = cs.pages()
    from_mask = []
    for p, words in zip(pages, mask):
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:p["count"]]
        from_mask.append(p["entities"][bits.astype(bool)])
    from_mask = np.sort(np.concatenate(from_mask))
    assert np.array_equal(from_mask, np.sort(res.ids.astype(np.int32)))


def test_empty_and_tiny(ctx, oracle):
    cs = lb.CullingSystem(ctx)
    f = lb.frustum_perspective(**scenes.c1_frustum_args())
    assert cs.cull(f).total == 0  # culling_system.cpp:322: no cells -> nothing
    cs.add(7, 2, (0.0, 0.0, -10.0), 1.0)
    r = cs.cull(f)
    assert r.total == 1 and r.ids[0] == 7 and r.types()[0] == 2
    cs.remove(7)
    assert cs.cull(f).total == 0


def test_tangent_and_border_cases(ctx, oracle):
    """Spheres within a few ulps of the planes, entities on cell borders and at negative coordinates (SURVEY §4 T2)."""
    rng = np.random.default_rng(21)
    args = scenes.c1_frustum_args()
    f = lb.frustum_perspective(**args)
    fb = lb.culling.frustum_bytes(f)
    xs, ys, zs, ds = (np.array(getattr(f, k)[:6], np.float64) for k in ("xs", "ys", "zs", "ds"))
    n = 40_000
    pos = (rng.random((n, 3)) * 2 - 1) * np.array([1800.0, 180.0, 1800.0])
    rad = (rng.random(n) * 4 + 0.5).astype(np.float32)
    # push each point onto a random plane at distance ~radius (tangent within rounding)
    k = rng.integers(0, 6, n)
    nrm = np.stack([xs[k], ys[k], zs[k]], axis=1)
    dist = (pos * nrm).sum(axis=1) + ds[k]
    pos = pos - nrm * (dist + rad.astype(np.float64))[:, None] + nrm * rng.normal(size=(n, 1)) * 1e-5
    # and a batch exactly on multiples of the cell size, incl. negative ones
    grid = (rng.integers(-6, 7, (5000, 3)) * 300.0).astype(np.float64)
    pos = np.concatenate([pos, grid])
    rad = np.concatenate([rad, np.full(5000, 2.0, np.float32)])
    scene = dict(entities=np.arange(len(pos), dtype=np.int32), types=np.zeros(len(pos), np.uint8), pos=pos, radius=rad)
    cs, oc = _both(ctx, oracle, scene)
    res = cs.cull(f)
    oids, otys, _ = oc.cull(fb)
    _assert_same(res, oids, otys)


def test_10m_properties(ctx):
    """Full C2 size: size-independent properties (the oracle is not run at this size inside the GPU suite)."""
    scene = scenes.c2_scene(10_000_000)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    r1 = cs.cull(f)
    r1.ids = r1.ids.copy()  # cull() returns a view of the result buffer, valid until the next cull
    # unique ids, all valid, type segments consistent with the scene's types
    assert len(np.unique(r1.ids)) == r1.total
    assert np.array_equal(scene["types"][r1.ids], r1.types())
    # idempotence + invariance to replica rotation
    r2 = cs.cull(f)
    assert np.array_equal(np.sort(r1.ids), np.sort(r2.ids))
    # per-type culls partition the all-types cull
    parts = [cs.cull(f, t).ids.copy() for t in range(4)]
    assert np.array_equal(np.sort(np.concatenate(parts)), np.sort(r1.ids))
    # a frustum containing the whole scene returns everything
    big = lb.frustum_ortho((0.0, 0.0, 20000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 20000.0, 20000.0, 0.0, 40000.0)
    assert cs.cull(big).total == 10_000_000


def test_c2_10m_equals_oracle_at_full_size(ctx, oracle):
    """BASELINE config[1] at its stated size: the sorted visible ids of every renderable type equal the oracle's (the oracle is pinned
    to the reference's compiled culling_system.cpp by tests/test_oracle_ref.py; bench.py repeats the digest against that build)."""
    scene = scenes.c2_scene(10_000_000)
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    res = cs.cull(f)
    oids, otys, st = oc.cull(lb.culling.frustum_bytes(f))
    assert res.total == len(oids) > 1_000_000
    got_t = res.types()
    for t in range(4):
        assert np.array_equal(np.sort(res.ids[got_t == t]), np.sort(oids[otys == t]).astype(res.ids.dtype)), f"type {t}"
    for k in ("pages_tested", "pages_inside", "pages_outside", "entities_tested"):
        assert res.stats[k] == st[k], k
    cs.close()


def test_special_radii_follow_the_reference(ctx):
    """NaN of either sign, infinities, -0.0, negative radii: movemask reads sign bits, and the reference's SSE subtraction hands a NaN
    radius through with the sign of -radius (tests/golden/cull_kat.npz: special_*, reference-run)."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "cull_kat.npz"))
    rad = g["special_radius_bits"].view(np.float32)
    n = len(rad)
    cs = lb.CullingSystem(ctx)
    cs.add(np.arange(n, dtype=np.int32), np.zeros(n, np.uint8), g["special_pos"], rad)
    res = cs.cull(lb.culling.frustum_from_bytes(g["frusta"][0]))
    got, exp = np.sort(res.ids).astype(np.int64), g["special_visible"].astype(np.int64)
    groups = ((0, 100, "+nan"), (100, 200, "-nan"), (200, 300, "+inf"), (300, 400, "-inf"), (400, 500, "-0.0"), (500, 600, "-3.5"), (600, n, "2.0"))
    summary = {name: (int(((got >= a) & (got < b)).sum()), int(((exp >= a) & (exp < b)).sum())) for a, b, name in groups}
    assert np.array_equal(got, exp), f"visible per radius class (got, reference): {summary}"
    cs.close()


def test_far_from_world_origin_and_negative_radius(ctx, oracle):
    """World coordinates of several thousand km (fp64 positions, fp32 cell-relative spheres) and a few negative radii
    (which switch the plane-masking shortcut off): visibility stays bit-exact."""
    rng = np.random.default_rng(77)
    n = 120_000
    base = np.array([3.0e6 + 17.25, -2.0e5 + 0.5, -7.5e6 + 3.125])
    pos = base + (rng.random((n, 3)) * 2 - 1) * np.array([2500.0, 250.0, 2500.0])
    rad = (rng.random(n) * 6 + 0.25).astype(np.float32)
    scene = dict(entities=np.arange(n, dtype=np.int32), types=(np.arange(n) % 2).astype(np.uint8), pos=pos, radius=rad)
    cs, oc = _both(ctx, oracle, scene)
    for d, far in (((0.0, 0.0, -1.0), 1500.0), ((0.6, -0.1, 0.79), 3000.0), ((-1.0, 0.02, 0.01), 800.0)):
        a = dict(scenes.c1_frustum_args(), position=tuple(base + np.array([100.0, 10.0, -50.0])), direction=d, far=far)
        f = lb.frustum_perspective(**a)
        res = cs.cull(f)
        oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
        _assert_same(res, oids, otys)
        assert res.total > 100
    # negative radii: plane masking must switch itself off and results stay identical to the reference arithmetic
    neg = rng.choice(n, 200, replace=False).astype(np.int32)
    nr = -(rng.random(200) * 50).astype(np.float32)
    cs.setRadius(neg, nr); oc.set_radius(neg, nr)
    f = lb.frustum_perspective(**dict(scenes.c1_frustum_args(), position=tuple(base), far=2500.0))
    res = cs.cull(f)
    oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
    _assert_same(res, oids, otys)


def test_overlapped_views_keep_results_apart(ctx, oracle):
    """cull_device_n issues independent culls on several streams / output lanes (and with programmatic dependent launch); whatever
    overlaps, the cull issued last must read exactly like a lone cull, also when single culls and batches interleave."""
    scene = scenes.cull_scene(400_000, (3000.0, 300.0, 3000.0), seed=31, big_fraction=0.004, type_probs=(0.7, 0.2, 0.1))
    cs, oc = _both(ctx, oracle, scene)
    a = scenes.c1_frustum_args()
    views = [lb.frustum_perspective(**dict(a, far=2500.0)),
             lb.frustum_perspective(**dict(a, position=(800.0, 0.0, 900.0), direction=(-0.5, 0.0, -0.8), far=1700.0)),
             lb.frustum_ortho((0.0, 0.0, 4000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 3000.0, 3000.0, 0.0, 8000.0)]
    base = np.concatenate([[0], np.cumsum(np.bincount(scene["types"], minlength=256))])

    def check_last(f):
        ptr, res = cs.last_result()
        oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
        assert res.total == len(oids) > 0
        for t in range(3):
            got = ctx.copy_to_host(ptr + 4 * int(base[t]), int(res.type_count[t]), np.uint32)
            assert np.array_equal(np.sort(got).astype(np.int64), np.sort(oids[otys == t]).astype(np.int64))
        bits = cs.read_bitmask()
        assert int(np.unpackbits(bits.view(np.uint8)).sum()) == len(oids)

    for n in (1, 2, 3, 4, 7, 16):
        for f in views:
            cs.cull_device_n(f, n)
            check_last(f)
    # batches of different views back to back, nothing read in between; then a single cull right behind a batch
    cs.cull_device_n(views[0], 5)
    cs.cull_device_n(views[2], 4)
    cs.cull_device_n(views[1], 3)
    check_last(views[1])
    cs.cull_device_n(views[2], 6)
    cs.cull_device(views[0], want_counts=False)
    check_last(views[0])
    assert np.array_equal(np.sort(cs.cull(views[2]).ids), np.sort(oc.cull(lb.culling.frustum_bytes(views[2]))[0]).astype(np.uint32))
    # an edit between batches goes through the context stream before the lanes fork
    moved = scene["entities"][:5000]
    newpos = scene["pos"][:5000] + np.array([40.0, 0.0, -25.0])
    cs.set(moved, newpos, scene["radius"][:5000])
    oc.set(moved, newpos, scene["radius"][:5000])
    cs.cull_device_n(views[0], 5)
    check_last(views[0])
    cs.close()


def test_pinned_and_pageable_destinations_agree(ctx, oracle):
    """lb200_culling_cull writes straight into a page-locked destination from the device and falls back to copies for pageable
    memory; both must hand back the oracle's sets, per type, and report the same counts; a too-small buffer is LB200_ERR_CAPACITY."""
    import ctypes as C
    from lumixengine_b200 import _lib
    scene = scenes.cull_scene(150_000, (3000.0, 300.0, 3000.0), seed=41, big_fraction=0.003, type_probs=(0.5, 0.3, 0.2))
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_perspective(**dict(scenes.c1_frustum_args(), far=2200.0))
    oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
    pinned = cs.cull(f)
    _assert_same(pinned, oids, otys)
    pageable = np.zeros(cs.entity_count(), np.uint32)  # plain numpy memory
    res = _lib.CullResult()
    rc = cs.L.lb200_culling_cull(cs.h, C.byref(f), C.c_uint8(0xFF), pageable.ctypes.data_as(C.c_void_p), C.c_uint32(len(pageable)), C.byref(res))
    assert rc == 0 and res.total == pinned.total
    assert list(res.type_count[:4]) == [int((otys == t).sum()) for t in range(4)]
    for t in range(3):
        o, c = int(res.type_offset[t]), int(res.type_count[t])
        assert np.array_equal(np.sort(pageable[o:o + c]).astype(np.int64), np.sort(oids[otys == t]).astype(np.int64))
        assert np.array_equal(np.sort(pinned.of_type(t)).astype(np.int64), np.sort(oids[otys == t]).astype(np.int64))
    small = ctx.host_alloc(16, np.uint32)
    rc = cs.L.lb200_culling_cull(cs.h, C.byref(f), C.c_uint8(0xFF), small.ctypes.data_as(C.c_void_p), C.c_uint32(16), C.byref(res))
    assert rc == _lib.ERR_CAPACITY and res.total == pinned.total
    cs.close()


def test_begin_poll_end_equals_cull(ctx, oracle):
    """The non-blocking delivery (what the engine shim uses from job fibers: begin, yield while poll is false, end) hands back exactly
    what cull() does, for a full cull and for one renderable type."""
    scene = scenes.cull_scene(200_000, (3000.0, 300.0, 3000.0), seed=51, big_fraction=0.004, type_probs=(0.6, 0.3, 0.1))
    cs, oc = _both(ctx, oracle, scene)
    f = lb.frustum_perspective(**dict(scenes.c1_frustum_args(), far=2400.0))
    for t in (lb.culling.TYPE_ALL, 1):
        oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f), -1 if t == lb.culling.TYPE_ALL else t)
        cs.cull_begin(f, t)
        spins = 0
        while not cs.cull_poll():
            spins += 1
            assert spins < 10_000_000
        res = cs.cull_end()
        _assert_same(res, oids, otys)
        _assert_same(cs.cull(f, t), oids, otys)
    cs.close()


def test_random_views_and_edits(ctx, oracle):
    """Randomised parity run (the same generator the oracle itself is checked with against the reference build in
    tests/test_oracle_ref.py): worlds with crowded and sparse cells, perspective / ortho views incl. axis-aligned ones snapped to cell
    corners, tiny and huge far planes, type filters, and batches of moves / radius changes / removals between the views."""
    rng = np.random.default_rng(2024)
    for world in range(3):
        n = int(rng.integers(2_000, 30_000))
        half = (float(rng.choice([250.0, 900.0, 4000.0])), float(rng.choice([50.0, 400.0])), float(rng.choice([250.0, 900.0, 4000.0])))
        scene = scenes.cull_scene(n, half, seed=300 + world, big_fraction=float(rng.choice([0.0, 0.02, 0.3])), type_probs=(0.5, 0.25, 0.25))
        cs, oc = _both(ctx, oracle, scene)
        alive = np.ones(n, bool)
        pos, rad = scene["pos"].copy(), scene["radius"].copy()
        for step in range(12):
            p = rng.normal(size=3) * np.array(half) * 1.5
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            up = np.cross(np.cross(d, rng.normal(size=3)), d); up /= np.linalg.norm(up)
            if step % 5 == 0:
                p = np.round(p / 300.0) * 300.0
                d, up = np.array([0.0, 0.0, -1.0]), np.array([0.0, 1.0, 0.0])
            far = float(rng.choice([30.0, 700.0, 5000.0, 60000.0]))
            if step % 3 == 2:
                f = lb.frustum_ortho(p, d.astype(np.float32), up.astype(np.float32), float(rng.uniform(10, 3000)), float(rng.uniform(10, 3000)), 0.0, far)
            else:
                f = lb.frustum_perspective(p, d.astype(np.float32), up.astype(np.float32), float(rng.uniform(0.2, 2.4)), float(rng.uniform(0.5, 2.5)),
                                           float(rng.uniform(0.01, 2.0)), far)
            t = int(rng.choice([-1, -1, 0, 1, 2]))
            oids, otys, st = oc.cull(lb.culling.frustum_bytes(f), t)
            res = cs.cull(f) if t < 0 else cs.cull(f, t)
            _assert_same(res, oids, otys)
            assert res.stats["pages_tested"] == st["pages_tested"] and res.stats["pages_inside"] == st["pages_inside"], (world, step)
            live = np.nonzero(alive)[0]
            mv = rng.choice(live, min(len(live), 400), replace=False).astype(np.int32)
            a, b, c = np.array_split(mv, 3)
            pos[a] = pos[a] + rng.normal(size=(len(a), 3)) * 200.0
            cs.setPosition(a, pos[a]); oc.set_position(a, pos[a])
            rad[b] = (rng.random(len(b)) * 500.0).astype(np.float32)
            cs.setRadius(b, rad[b]); oc.set_radius(b, rad[b])
            cs.remove(c); oc.remove(c)
            alive[c] = False
        cs.close()


def _canon(res):
    return np.sort(res.ids.astype(np.int64) * 256 + res.types())


def test_device_rebinning_equals_host_set(ctx, oracle):
    """SURVEY 8f N3: CullingSystem::set for a batch of movers on the device (in-cell overwrites, cell / big-ness changers through tombstones,
    page compaction, the sorted re-insertion) against the oracle's sequential set(): same visible sets for several views, frame after frame,
    and the host mirror pulled back from the device agrees entity by entity."""
    rng = np.random.default_rng(21)
    n = 150_000
    scene = scenes.cull_scene(n, (3000.0, 300.0, 3000.0), seed=5, big_fraction=0.01, type_probs=(0.7, 0.2, 0.1))
    cs, oc = _both(ctx, oracle, scene)
    a = scenes.c1_frustum_args()
    views = [lb.frustum_perspective(**dict(a, far=3000.0)), lb.frustum_perspective(**dict(a, position=(700.0, 20.0, -400.0), direction=(-0.7, -0.05, 0.7), far=2500.0)),
             lb.frustum_ortho((0.0, 0.0, 5000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 5000.0, 5000.0, 0.0, 10000.0)]
    pos, rad = scene["pos"].copy(), scene["radius"].copy()
    for frame in range(4):
        if frame < 3:  # every entity moves: most stay in their cell, some cross borders, some change big-ness, a crowd teleports into one cell
            pos = pos + rng.normal(size=pos.shape) * np.array([25.0, 3.0, 25.0])
            rad = np.where(rng.random(n) < 0.02, (rng.random(n) * 650).astype(np.float32), rad).astype(np.float32)
            if frame == 1:
                crowd = rng.choice(n, 4000, replace=False)
                pos[crowd] = np.array([1234.0, 10.0, -777.0]) + rng.random((4000, 3)) * 40.0
            ents = np.arange(n, dtype=np.int32)
            d_pos, d_rad = ctx.to_device(pos), ctx.to_device(rad)
            changers = cs.set_many_device(d_pos, d_rad, n)
            ctx.free_device(d_pos); ctx.free_device(d_rad)
            assert changers > 100
        else:  # a subset given by an id list, after host-side edits in between (the host mirror is pulled back, edited, pushed again)
            gone = rng.choice(n, 500, replace=False).astype(np.int32)
            cs.remove(gone); oc.remove(gone)
            ents = np.setdiff1d(rng.choice(n, 30_000, replace=False), gone).astype(np.int32)
            pos[ents] += rng.normal(size=(len(ents), 3)) * np.array([200.0, 10.0, 200.0])
            d_ents, d_pos, d_rad = ctx.to_device(ents), ctx.to_device(pos[ents]), ctx.to_device(rad[ents])
            cs.set_many_device(d_pos, d_rad, len(ents), dev_entities=d_ents, max_entity=n - 1)
            for p in (d_ents, d_pos, d_rad):
                ctx.free_device(p)
        oc.set(ents, pos[ents], rad[ents])
        for f in views:
            res = cs.cull(f)
            oi, ot, _ = oc.cull(lb.culling.frustum_bytes(f))
            assert res.total == len(oi) and np.array_equal(_canon(res), np.sort(oi.astype(np.int64) * 256 + ot)), f"frame {frame}"
        if frame in (1, 3):  # host mirror after the pull-back: every entity in the cell of its position, sphere relative to the page origin
            cs.sync_host()
            assert cs.page_count() > 0
            seen = np.zeros(n, bool)
            for pg in cs.pages():
                e = pg["entities"]
                assert pg["count"] == len(e) <= 200 and not seen[e].any()
                seen[e] = True
                key = (pos[e] * np.float32(1 / 300.0)).astype(np.int64)  # trunc toward zero like IVec3(DVec3)
                assert np.all(key == np.asarray(pg["indices"])[None, :]) and np.all((rad[e] > 300.0) == bool(pg["is_big"]))
                assert np.array_equal(pg["spheres"][:, :3], (pos[e] - np.asarray(pg["origin"])).astype(np.float32)) and np.array_equal(pg["spheres"][:, 3], rad[e])
            alive = np.ones(n, bool)
            if frame == 3:
                alive[gone] = False
            assert np.array_equal(seen, alive)
    cs.close()


def test_const_getters_pull_back_the_device_state(ctx, oracle):
    """The four const getters of the C API read the host mirror.  Each one, called first after a device re-binning batch (no
    sync_host), pulls the device state back itself: it answers for the batch, and the mirror it leaves agrees entity by entity."""
    import ctypes as C
    from lumixengine_b200 import _lib
    rng = np.random.default_rng(77)
    n = 30_000
    scene = scenes.cull_scene(n, (2000.0, 300.0, 2000.0), seed=17, big_fraction=0.01, type_probs=(0.7, 0.2, 0.1))
    cs, _ = _both(ctx, oracle, scene)
    pos, rad = scene["pos"].copy(), scene["radius"].copy()

    def batch(crowd=0):  # every entity moves, some change their radius (and big-ness); the device is ahead of the mirror afterwards
        nonlocal pos, rad
        pos = pos + rng.normal(size=pos.shape) * np.array([60.0, 3.0, 60.0])
        c = rng.choice(n, crowd, replace=False)  # teleported into an empty cell far outside the scene: new pages
        pos[c] = np.array([6100.0, 10.0, 6100.0]) + rng.random((crowd, 3)) * 40.0
        changed = rng.random(n) < 0.05
        rad = np.where(changed, (rng.random(n) * 650).astype(np.float32), rad).astype(np.float32)
        d_pos, d_rad = ctx.to_device(pos), ctx.to_device(rad)
        assert cs.set_many_device(d_pos, d_rad, n) > 100
        ctx.free_device(d_pos); ctx.free_device(d_rad)
        return np.nonzero(changed)[0]

    def check_page(origin, indices, is_big, spheres, e):
        key = (pos[e] * np.float32(1 / 300.0)).astype(np.int64)  # trunc toward zero like IVec3(DVec3)
        assert np.all(key == np.asarray(indices)[None, :]) and np.all((rad[e] > 300.0) == bool(is_big))
        assert np.array_equal(spheres[:, :3], (pos[e] - np.asarray(origin)).astype(np.float32)) and np.array_equal(spheres[:, 3], rad[e])

    def check_mirror():
        seen = np.zeros(n, bool)
        for pg in cs.pages():
            e = pg["entities"]
            assert pg["count"] == len(e) <= 200 and not seen[e].any()
            seen[e] = True
            check_page(pg["origin"], pg["indices"], pg["is_big"], pg["spheres"], e)
        assert seen.all()
        return len(cs.pages())

    changed = batch()
    radii = [cs.L.lb200_culling_get_radius(cs.h, C.c_int32(int(e))) for e in changed[:50]]
    assert np.array_equal(np.array(radii, np.float32), rad[changed[:50]])
    before = check_mirror()

    batch(crowd=6000)
    count = int(cs.L.lb200_culling_page_count(cs.h))
    cs.sync_host()  # a no-op unless page_count left the device ahead: the references below do not go through page_count's pull-back
    assert count > before and count == int(cs.L.lb200_culling_page_count(cs.h)) == check_mirror()

    batch()
    o, ind = (C.c_double * 3)(), (C.c_int32 * 3)()
    ty, big, cnt = C.c_uint8(), C.c_uint8(), C.c_uint32()
    sph = np.empty((_lib.PAGE_SLOTS, 4), np.float32)
    ent = np.empty(_lib.PAGE_SLOTS, np.int32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    rc = cs.L.lb200_culling_get_page(cs.h, C.c_uint32(0), o, ind, C.byref(ty), C.byref(big), C.byref(cnt), ptr(sph), ptr(ent))
    assert rc == 0 and cnt.value > 0
    check_page(tuple(o), tuple(ind), big.value, sph[:cnt.value], ent[:cnt.value])
    check_mirror()

    batch()
    ids = []
    while (p := int(cs.L.lb200_culling_page_id(cs.h, C.c_uint32(len(ids))))) >= 0:
        ids.append(p)
    assert np.array_equal(np.array(ids, np.int64), cs.page_ids())
    check_mirror()
    cs.close()


def test_buffers_grow_after_first_use(ctx, oracle):
    """Every buffer that grows on demand is re-allocated after its first use, and the results stay equal to the oracle's: more entities
    than the page arrays and the output ids were sized for, a sparse upload of more pages than the first one staged, and a device
    re-binning batch with more movers, entities and pages than the first batch."""
    rng = np.random.default_rng(44)
    n, n0 = 200_000, 20_000
    scene = scenes.cull_scene(n, (30000.0, 300.0, 30000.0), seed=61, type_probs=(0.7, 0.2, 0.1))
    pos, rad = scene["pos"].copy(), scene["radius"].copy()
    cs = lb.CullingSystem(ctx)
    oc = oracle.OracleCulling()
    a = scenes.c1_frustum_args()
    views = [lb.frustum_perspective(**dict(a, far=20000.0)), lb.frustum_ortho((0.0, 0.0, 40000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 40000.0, 40000.0, 0.0, 80000.0)]

    def check(step):
        for f in views:
            res = cs.cull(f)
            oi, ot, _ = oc.cull(lb.culling.frustum_bytes(f))
            assert res.total == len(oi) and np.array_equal(_canon(res), np.sort(oi.astype(np.int64) * 256 + ot)), step

    def move(ids, sigma):
        pos[ids] += rng.normal(size=(len(ids), 3)) * np.array([sigma, 1.0, sigma])
        cs.setPosition(ids, pos[ids]); oc.set_position(ids, pos[ids])

    def rebin(ids, max_entity):
        pos[ids] += rng.normal(size=(len(ids), 3)) * np.array([400.0, 10.0, 400.0])
        d_ents, d_pos, d_rad = ctx.to_device(ids), ctx.to_device(pos[ids]), ctx.to_device(rad[ids])
        cs.set_many_device(d_pos, d_rad, len(ids), dev_entities=d_ents, max_entity=max_entity)
        for p in (d_ents, d_pos, d_rad):
            ctx.free_device(p)
        oc.set(ids, pos[ids], rad[ids])

    def add(lo, hi):
        s = slice(lo, hi)
        cs.add(scene["entities"][s], scene["types"][s], pos[s], rad[s]); oc.add(scene["entities"][s], scene["types"][s], pos[s], rad[s])

    add(0, n0)
    check("first upload")
    move(rng.choice(n0, 10, replace=False).astype(np.int32), 50.0)  # a sparse upload of a few pages
    check("small sparse upload")
    rebin(rng.choice(n0, 1000, replace=False).astype(np.int32), n0 - 1)
    check("small re-binning batch")
    add(n0, n)  # ten times the entities: the page arrays and output ids grow
    check("grown scene")
    assert cs.page_count() > 8 * 2 * 800
    move(rng.choice(n, 800, replace=False).astype(np.int32), 50.0)  # still a sparse upload, of more pages than the first one
    check("large sparse upload")
    rebin(rng.permutation(n).astype(np.int32), n - 1)  # more movers, entities and pages than the first batch
    check("large re-binning batch")
    cs.close()
