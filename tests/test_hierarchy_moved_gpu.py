"""The moved list of a hierarchy propagate (Hierarchy.markMoved / setEntities / propagateMoved, lb200_hierarchy_propagate_moved): the
entities whose `transformed` delegates World::transformEntity (world.cpp:255-282) fires, handed out on the device.

The list is held to `moved_closure` below, which restates the reference's recursion (each marked entity, then its children through
first_child / next_sibling, recursively), and, where oracle/_ref/libengine_shim_b200.so was built, to the delegates the reference's own World
fires for the same root moves.  Globals are held to plain propagate on a twin hierarchy and to the oracle bit for bit, spheres to
refresh_spheres bit for bit, and the chain propagateMoved -> onModelInstanceMoved -> CullingSystem::set -> cull -> createSortKeys ->
endFrame to the oracle in which only the closure is MOVED and re-set.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes, sortkeys
from lumixengine_b200._lib import LumixB200Error

pytestmark = pytest.mark.gpu
SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libengine_shim_b200.so")
FIELDS = ("pos", "rot", "scale")


def moved_closure(parents, marked, entity_of_node):
    """world.cpp:255-282: transformEntity(e) fires e's delegates, then recurses into every child (first_child / next_sibling, world.h:157-164,
    built as setParent builds them, world.cpp:672-676).  -> sorted entity ids whose delegates fire (entity -1: no listener)."""
    n = len(parents)
    first_child = [-1] * n
    next_sibling = [-1] * n
    for i in range(n):
        p = int(parents[i])
        if p >= 0:
            next_sibling[i] = first_child[p]
            first_child[p] = i
    fired = set()
    for m in marked:
        stack = [int(m)]
        while stack:
            e = stack.pop()
            if entity_of_node[e] >= 0:
                fired.add(int(entity_of_node[e]))
            c = first_child[e]
            while c >= 0:
                stack.append(c)
                c = next_sibling[c]
    return np.array(sorted(fired), np.int64)


def _as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)


def _random_transforms(rng, k, extent=500.0):
    t = np.zeros(k, lb.TRANSFORM_DTYPE)
    t["pos"] = (rng.random((k, 3)) * 2.0 - 1.0) * extent
    t["rot"] = scenes.random_unit_quats(rng, k)
    t["scale"] = (0.7 + 0.6 * rng.random((k, 3))).astype(np.float32)
    return t


def _bits_equal(a, b, what):
    for f in FIELDS:
        assert np.ascontiguousarray(a[f]).tobytes() == np.ascontiguousarray(b[f]).tobytes(), f"{what}: {f} differs"


def _read(ctx, ml):
    """Host copies of a MovedList: (entities, transforms, pos3 or None, radius or None)."""
    k = ml.count
    if k == 0:
        return np.zeros(0, np.int32), np.zeros(0, lb.TRANSFORM_DTYPE), None, None
    ent = ctx.copy_to_host(ml.entities, k, np.int32)
    tr = ctx.copy_to_host(ml.transforms, k, lb.TRANSFORM_DTYPE)
    pos = ctx.copy_to_host(ml.pos3, 3 * k, np.float64).reshape(k, 3) if ml.pos3 else None
    rad = ctx.copy_to_host(ml.radius, k, np.float32) if ml.radius else None
    return ent, tr, pos, rad


# ------------------------------------------------------------------------------------------------------------------------ topologies
def _chain(depth, width=1):
    """`width` chains of `depth` nodes, node k + width under node k."""
    p = np.full(depth * width, -1, np.int32)
    p[width:] = np.arange(width * (depth - 1), dtype=np.int32)
    return p


def _star(children, grandchildren=64):
    """One root with `children` children (one level past or at SMALL_LEVEL_NODES), a few of them with a child each, and a second root."""
    p = np.full(children + grandchildren + 2, -1, np.int32)
    p[1:children + 1] = 0
    p[children + 1:children + 1 + grandchildren] = np.arange(1, grandchildren + 1, dtype=np.int32) * 7
    return p


def _shuffled_forest(n, depth, fanout, seed):
    """hierarchy_forest with its nodes permuted: children come before their parents, level order is not node order."""
    parents, _, _ = scenes.hierarchy_forest(n, depth, fanout, seed=seed)
    perm = np.random.default_rng(seed).permutation(len(parents))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    return np.where(parents[perm] >= 0, inv[np.maximum(parents[perm], 0)], -1).astype(np.int32)


def _random_roots(n, roots, seed):
    """Several roots, random trees: node i >= roots hangs under a random earlier node."""
    rng = np.random.default_rng(seed)
    p = np.full(n, -1, np.int32)
    p[roots:] = (rng.random(n - roots) * np.arange(roots, n)).astype(np.int32)
    return p


TOPOLOGIES = {
    "forest": lambda: _shuffled_forest(20_000, 6, 4, seed=5),
    "chain_300": lambda: _chain(300, 3),             # past the 30 levels propagate_small_levels_kernel takes
    "chain_30": lambda: _chain(31, 5),               # 30 levels below the roots: all of them in the small-levels kernel
    "chain_32": lambda: _chain(32, 5),               # one level past them
    "star_8192": lambda: _star(8192),                # a level of SMALL_LEVEL_NODES: still the small-levels kernel
    "star_8193": lambda: _star(8193),                # one node more: the per-level kernel
    "roots": lambda: _random_roots(6000, 40, seed=8),
}


def _children(parents):
    n = len(parents)
    has_child = np.zeros(n, bool)
    has_child[parents[parents >= 0]] = True
    return has_child


def _mark_cases(parents, rng):
    """(name, marked nodes): none, a leaf, an inner node, a root, a node together with an ancestor, everything, 3 % at random."""
    has_child = _children(parents)
    leaves = np.nonzero(~has_child)[0]
    inner = np.nonzero(has_child & (parents >= 0))[0]
    roots = np.nonzero((parents < 0) & has_child)[0]
    x = int(rng.choice(np.nonzero(parents >= 0)[0]))
    anc = _root_of(parents, x)
    cases = [("none", []), ("leaf", [int(rng.choice(leaves))]), ("root", [int(rng.choice(roots))]),
             ("node and ancestor", [x, anc, x]), ("everything", list(range(len(parents)))),
             ("random", rng.choice(len(parents), max(1, len(parents) // 33), replace=False).tolist())]
    if len(inner):
        cases.insert(2, ("inner", [int(rng.choice(inner))]))
    return cases


def _root_of(parents, i):
    while parents[i] >= 0:
        i = int(parents[i])
    return i


def _setup(ctx, parents, seed):
    rng = np.random.default_rng(seed)
    n = len(parents)
    locals_ = _random_transforms(rng, n, 10.0)
    roots = _random_transforms(rng, n, 2000.0)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    return h, locals_, roots


# ------------------------------------------------------------------------------------------------------------------------ 1 + 2 + 6
@pytest.mark.parametrize("topology", list(TOPOLOGIES))
def test_moved_list_is_the_closure_and_outputs_match(ctx, oracle, topology):
    """Every mark case on every topology (both propagate kernels, levels of 8192 / 8193 nodes, depths 31 / 32 / 300): the list equals the
    closure, in ascending node index; globals equal plain propagate on a twin and the oracle; listed transforms equal those globals; spheres
    equal refresh_spheres' entries bit for bit."""
    parents = TOPOLOGIES[topology]()
    n = len(parents)
    rng = np.random.default_rng(n)
    h, locals_, roots = _setup(ctx, parents, seed=n + 1)
    twin, _, _ = _setup(ctx, parents, seed=n + 1)
    entity = np.where(rng.random(n) < 0.8, rng.permutation(n) + 3, -1).astype(np.int32)  # a non-identity map with -1 entries
    h.setEntities(entity)
    br = (0.5 + 2.5 * rng.random(n)).astype(np.float32)
    first = True
    for name, marked in _mark_cases(parents, rng):
        # the root case moves roots through setSubset(globals), the inner / leaf cases change locals through setSubset: both forms mark
        if name == "root":
            vals = _random_transforms(rng, len(marked), 2000.0)
            for x in (h, twin):
                x.setSubset(marked, vals, globals_=True)
            roots[marked] = vals
        elif name in ("inner", "leaf"):
            vals = _random_transforms(rng, len(marked), 10.0)
            for x in (h, twin):
                x.setSubset(marked, vals)
            locals_[marked] = vals
        else:
            h.markMoved(marked)
        ml = h.propagateMoved(br if first else None)
        first = False
        twin.propagate()
        want = moved_closure(parents, marked, entity)
        ent, tr, pos, rad = _read(ctx, ml)
        assert ml.count == len(want), f"{topology} / {name}: {ml.count} listed, the closure has {len(want)}"
        assert np.array_equal(np.sort(ent), want), f"{topology} / {name}: other entities than the closure"
        nodes = np.nonzero(np.isin(entity, want))[0]  # ascending node index
        assert np.array_equal(ent, entity[nodes]), f"{topology} / {name}: not in ascending node index"
        g = h.getTransforms()
        _bits_equal(g, twin.getTransforms(), f"{topology} / {name}: propagate_moved against propagate")
        if name in ("none", "root", "everything"):
            exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
            _bits_equal(g, exp, f"{topology} / {name}: against the oracle")
        _bits_equal(tr, g[nodes], f"{topology} / {name}: listed transforms")
        d_pos, d_rad = twin.refreshSpheres(br)
        all_pos = ctx.copy_to_host(d_pos, 3 * n, np.float64).reshape(n, 3)
        all_rad = ctx.copy_to_host(d_rad, n, np.float32)
        if len(nodes):
            assert pos.tobytes() == all_pos[nodes].tobytes() and rad.tobytes() == all_rad[nodes].tobytes(), f"{topology} / {name}: spheres"
        if name == "everything":
            assert len(nodes) == (entity >= 0).sum()
    h.close()
    twin.close()


# ------------------------------------------------------------------------------------------------------------------------ reference World
@pytest.fixture(scope="module")
def shim():
    if not os.path.exists(SO):
        pytest.skip("oracle/_ref/libengine_shim_b200.so not built (needs /root/reference at build time)")
    L = C.CDLL(SO)
    os.environ["LB200_ENGINE_SHIM_LOADED"] = "1"  # the engine's job system cannot be shut down on Linux: tests/conftest.py leaves with os._exit
    L.wshim_run.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("topology", ["forest", "chain_300", "star_8193", "roots"])
def test_moved_list_is_what_the_reference_world_fires(ctx, shim, topology):
    """Root moves (what the World shim moves): the entities whose `transformed` delegates the reference's own World fires in one round of
    World::setTransform are exactly the moved list, listens = entity != -1; the World binding (World::propagateHierarchyB200 over the moved
    list) fires the same delegates the same number of times.  No roots, one root, half the roots, every root (every node listed)."""
    parents = TOPOLOGIES[topology]()
    n = len(parents)
    rng = np.random.default_rng(n + 7)
    _, locals_, roots = scenes.hierarchy_forest(n, 2, 2, seed=n)
    listens = (rng.random(n) < 0.7).astype(np.uint8)
    entity = np.where(listens == 1, np.arange(n), -1).astype(np.int32)
    h = lb.Hierarchy(ctx, parents)
    h.setEntities(entity)
    root_ids = np.nonzero(parents < 0)[0].astype(np.uint32)
    for moved in (root_ids[:0], root_ids[:1], rng.choice(root_ids, max(1, len(root_ids) // 2), replace=False).astype(np.uint32), root_ids):
        vals = _random_transforms(rng, len(moved), 300.0)
        out_ref, out_b = np.zeros(n, lb.TRANSFORM_DTYPE), np.zeros(n, lb.TRANSFORM_DTYPE)
        calls_ref, calls_b = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        seconds = np.zeros(2)
        rc = shim.wshim_run(_p(parents), _p(np.ascontiguousarray(locals_)), _p(np.ascontiguousarray(roots)), C.c_uint32(n), _p(listens),
                            _p(np.ascontiguousarray(moved)), _p(np.ascontiguousarray(vals)), C.c_uint32(len(moved)), C.c_uint32(1), C.c_int(0),
                            _p(out_ref), _p(out_b), _p(calls_ref), _p(calls_b), _p(seconds), None)
        assert rc == 0
        fired = np.nonzero(calls_ref)[0]
        assert (calls_ref <= 1).all()
        h.markMoved(moved)
        ml = h.propagateMoved()
        ent, _, _, _ = _read(ctx, ml)
        assert np.array_equal(np.sort(ent), fired), f"{topology}, {len(moved)} roots moved: the reference World fired other delegates"
        assert np.array_equal(fired, moved_closure(parents, moved, entity))
        assert np.array_equal(calls_b, calls_ref), f"{topology}, {len(moved)} roots moved: the World binding fired other delegates"
        for f in FIELDS:
            assert out_ref[f].tobytes() == out_b[f].tobytes()
    h.close()


# ------------------------------------------------------------------------------------------------------------------------ 3: marks
def test_mark_lifecycle(ctx):
    parents = _shuffled_forest(5000, 5, 3, seed=11)
    n = len(parents)
    rng = np.random.default_rng(3)
    h, locals_, roots = _setup(ctx, parents, seed=12)
    ident = np.arange(n, dtype=np.int32)
    listed = lambda ml: np.sort(_read(ctx, ml)[0])  # noqa: E731
    assert h.propagateMoved().count == 0, "a new hierarchy has no marks"
    # whole-array uploads and compute_locals mark nothing
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.setTransforms(_random_transforms(rng, n))
    h.computeLocalTransforms()
    ml = h.propagateMoved()
    assert ml.count == 0 and ml.pos3 is None and ml.radius is None, "no radii held: no spheres"
    # both forms of setSubset mark
    x = int(np.nonzero(parents >= 0)[0][7])
    r = int(np.nonzero(parents < 0)[0][3])
    h.setSubset([x], _random_transforms(rng, 1, 10.0))
    h.setSubset([r], _random_transforms(rng, 1), globals_=True)
    assert np.array_equal(listed(h.propagateMoved()), moved_closure(parents, [x, r], ident))
    # plain propagate leaves the marks to the next propagateMoved; a second propagateMoved without edits lists nothing
    h.markMoved([x])
    h.propagate()
    h.propagate()
    assert np.array_equal(listed(h.propagateMoved()), moved_closure(parents, [x], ident))
    assert h.propagateMoved().count == 0
    # an out-of-range node is refused and marks nothing, also the valid nodes of the same call
    with pytest.raises(LumixB200Error):
        h.markMoved([x, n])
    assert h.propagateMoved().count == 0
    h.markMoved([])
    # without the count read-back the call does not wait: the count is in device memory
    h.markMoved([r])
    ml = h.propagateMoved(np.ones(n, np.float32), read_count=False)
    assert ml.count is None and ml.pos3 and ml.radius
    ctx.synchronize()
    assert int(ctx.copy_to_host(ml.count_ptr, 1, np.uint32)[0]) == len(moved_closure(parents, [r], ident))
    # the radii are held from now on
    h.markMoved([r])
    ml = h.propagateMoved()
    assert ml.pos3 and ml.radius
    h.close()


# ------------------------------------------------------------------------------------------------------------------------ 4: entity map
@pytest.mark.parametrize("device", [False, True])
def test_marks_and_entities_follow_their_nodes_across_set_parents(ctx, device):
    parents = _random_roots(3000, 12, seed=4)
    n = len(parents)
    rng = np.random.default_rng(9)
    h, _, _ = _setup(ctx, parents, seed=2)
    entity = np.where(rng.random(n) < 0.85, rng.permutation(n) + 100, -1).astype(np.int32)
    h.setEntities(entity)

    def set_parents(p):
        if device:
            d = ctx.to_device(np.ascontiguousarray(p, np.int32))
            h.setParentsDevice(d, len(p))
            ctx.free_device(d)
        else:
            h.setParents(p)

    def listed():
        ml = h.propagateMoved()
        return np.sort(_read(ctx, ml)[0])

    # re-parenting a marked subtree: the closure is taken over the new topology
    has_child = _children(parents)
    x = int(np.nonzero(has_child & (parents >= 0))[0][5])
    other = int(np.setdiff1d(np.nonzero(parents < 0)[0], [_root_of(parents, x)])[0])
    p2 = parents.copy()
    p2[x] = other
    h.markMoved([x])
    set_parents(p2)
    assert np.array_equal(listed(), moved_closure(p2, [x], entity))
    # an unmarked node's new parent is marked: the moved node comes along
    h.markMoved([other])
    assert np.array_equal(listed(), moved_closure(p2, [other], entity))
    # growing: old nodes keep marks and entity ids, new nodes start unmarked with entity i
    grow = 500
    p3 = np.concatenate([p2, (rng.random(grow) * n).astype(np.int32)])
    marked = [x, int(rng.choice(n))]
    h.markMoved(marked)
    set_parents(p3)
    ent3 = np.concatenate([entity, np.arange(n, n + grow, dtype=np.int32)])
    assert np.array_equal(listed(), moved_closure(p3, marked, ent3)), "new nodes under marked ones are listed, with entity i"
    h.markMoved([n + 10])
    assert np.array_equal(listed(), [n + 10])
    # shrinking: marks of dropped nodes are gone, the kept nodes keep theirs
    keep = 2000
    p4 = np.where(p3[:keep] < keep, p3[:keep], -1).astype(np.int32)
    dropped = int(np.nonzero(np.arange(len(p3)) >= keep)[0][0])
    kept = int(np.nonzero(p4 >= 0)[0][3])
    h.markMoved([dropped, kept])
    set_parents(p4)
    assert np.array_equal(listed(), moved_closure(p4, [kept], entity[:keep]))
    h.close()


# ------------------------------------------------------------------------------------------------------------------------ 5: device chain
LIGHT = (0.3, -0.8, 0.2)
CASCADES = (40.0, 200.0, 900.0, 2500.0)
SHADOW_BUCKETS = [0, 0xff, 0xff, 1]
INV_CELL = np.float64(np.float32(1 / 300.0))  # the culling system's IVec3(pos * (1 / 300.f))


def _cells(pos):
    return np.trunc(np.asarray(pos, np.float64) * INV_CELL).astype(np.int64)


def _canon(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare_view(got, exp, what):
    gk, gv = _canon(got["keys"], got["values"])
    ek, ev = _canon(exp["keys"], exp["values"])
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev), f"{what}: pairs differ ({len(gk)} against {len(ek)})"
    assert np.array_equal(got["group_count"], exp["group_count"]) and np.array_equal(got["group_offset"], exp["group_offset"]), what
    go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
    assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo]), what
    g_of = np.repeat(np.arange(len(exp["group_count"])), exp["group_count"])
    assert np.array_equal(g_of[go], g_of[eo]), what
    assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo]), what


def test_device_chain_moves_only_the_closure(ctx, oracle):
    """Config 3 (1 M nodes), three frames with about 1 % of the roots moved: setSubset -> propagateMoved -> moveDevice(list) ->
    set_many_device(list) -> cull_views (main view + cascades) -> createSortKeysViews -> endFrame, against the oracle in which only the
    closure is MOVED and re-set: visible sets, keys and values, groups with their instance data, prev_frame_transform, the changer count."""
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3, root_extent=(2500.0, 300.0, 2500.0))
    n = len(parents)
    rng = np.random.default_rng(17)
    entity = rng.permutation(n).astype(np.int32)  # node i is entity entity[i]
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.setEntities(entity)
    h.propagate()
    br = (0.5 + 2.5 * rng.random(n)).astype(np.float32)
    g = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    # per entity: transform and sphere
    tr_e = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr_e[entity] = g
    pos_e = np.zeros((n, 3))
    pos_e[entity] = g["pos"]
    rad_e = np.zeros(n, np.float32)
    rad_e[entity] = oracle.sphere_radius(_as_bytes(g), br)
    types = np.zeros(n, np.uint8)
    ents = np.arange(n, dtype=np.int32)
    cs = lb.CullingSystem(ctx)
    cs.add(ents, types, pos_e, rad_e)
    cs.set_replicas(1)
    oc = oracle.OracleCulling()
    oc.add(ents, types, pos_e, rad_e)
    sk = scenes.sortkey_setup(n, types, pos_e, seed=23, moved_fraction=0.0)
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(tr_e)
    lod, pf = sk["lod"].copy(), sk["pose_frame"].copy()
    prev_exp = np.zeros(n, lb.TRANSFORM_DTYPE)
    root_ids = np.nonzero(parents < 0)[0]
    big_roots = root_ids[_children(parents)[root_ids]]
    cam = dict(scenes.c1_frustum_args(), far=2500.0)
    args = [cam] + scenes.shadow_cascade_args(cam, LIGHT, CASCADES)
    frusta = [lb.frustum_perspective(**a) if "fov" in a else lb.frustum_ortho(**a) for a in args]
    for frame in range(3):
        moved = rng.choice(root_ids, len(root_ids) // 100, replace=False)
        moved = np.union1d(moved, big_roots[frame % len(big_roots)]).astype(np.uint32)  # one whole tree each frame
        vals = roots[moved].copy()
        vals["pos"] += rng.normal(size=(len(moved), 3)) * 400.0
        vals["rot"] = scenes.random_unit_quats(rng, len(moved))
        roots[moved] = vals
        # the device frame
        h.setSubset(moved, vals, globals_=True)
        ml = h.propagateMoved(br if frame == 0 else None)
        S.moveDevice(ml.entities, ml.transforms, ml.count)
        changers = cs.set_many_device(ml.pos3, ml.radius, ml.count, dev_entities=ml.entities, max_entity=n - 1)
        cs.cull_views(frusta, want_counts=False)
        views = [sortkeys.make_view(a["position"], cam["position"], 0.15, 1.25, 50 + frame, k > 0, sk["max_sort_key"],
                                    *((sk["layer_to_bucket"], sk["depth_sorted_buckets"]) if k == 0 else (SHADOW_BUCKETS, ())))
                 for k, a in enumerate(args)]
        res = S.createSortKeysViews(cs, views)
        got = [S.readView(k, r) for k, r in enumerate(res)]
        S.endFrame()
        prev = S.prevTransforms()
        # the oracle's frame: only the closure moves
        g = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
        closure = np.nonzero(np.isin(entity, moved_closure(parents, moved, entity)))[0]  # nodes, ascending
        ce = entity[closure]
        assert ml.count == len(closure) > len(moved)
        ent, tr, _, _ = _read(ctx, ml)
        assert np.array_equal(ent, ce)
        _bits_equal(tr, g[closure], f"frame {frame}: listed transforms")
        new_pos = np.ascontiguousarray(g["pos"][closure])
        new_rad = oracle.sphere_radius(_as_bytes(g[closure]), br[closure])
        exp_changers = int((np.any(_cells(pos_e[ce]) != _cells(new_pos), axis=1) | ((rad_e[ce] > 300.0) != (new_rad > 300.0))).sum())
        assert changers == exp_changers, f"frame {frame}: set_many_device reports {changers} changers, {exp_changers} movers changed cell or is_big"
        assert changers > 0
        oc.set(ce, new_pos, new_rad)
        pos_e[ce], rad_e[ce] = new_pos, new_rad
        tr_e[ce] = g[closure]
        flags = sk["flags"].copy()
        flags[ce] |= sortkeys.MOVED
        moved_visible = 0
        for v, (f, view) in enumerate(zip(frusta, views)):
            oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
            exp = oracle.create_sort_keys(oids, otys, tr_e, sk["model_of"], lod, flags, pf, sk["decal_sort_key"], sk["decal_layer"],
                                          sk["models"], sk["meshes"], view)
            assert res[v].n_keys == len(exp["keys"]), f"frame {frame} view {v}"
            _compare_view(got[v], exp, f"frame {frame} view {v}")
            moved_visible += int(np.isin(ce, oids).sum())
        assert moved_visible > 0, "moved instances should be in view"
        assert np.array_equal(got[0]["lod"][:n].view(np.uint32), lod.view(np.uint32))
        prev_exp[ce] = tr_e[ce]
        _bits_equal(prev, prev_exp, f"frame {frame}: prev_frame_transform")
    S.close()
    cs.close()
    h.close()
