"""Topology changes on the device: lb200_hierarchy_set_parents / _set_parents_device against the level order the host BFS built before
the builder moved to the device (restated here in numpy), and against the oracle for everything computed on the new level order.

The level order: level 0 = the roots in ascending node index; level l + 1 = the children of level l's nodes, walked in level order, each
node's children in ascending node index.  parent_pos = the parent's level position.  Node i < min(old n, new n) keeps its transforms across
a re-parent; nodes new to the hierarchy start as the identity.  Every comparison is bit for bit.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes
from bitexact import assert_bits_equal, assert_transforms_equal

pytestmark = pytest.mark.gpu

GRIDS = (1, 2, 3, 0)  # max_blocks of the builder's cooperative kernels; 0 = every co-resident block


def _as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)


def _transforms(rng, n, extent):
    t = np.zeros(n, lb.TRANSFORM_DTYPE)
    t["pos"] = (rng.random((n, 3)) * 2.0 - 1.0) * np.asarray(extent, np.float64)
    t["rot"] = scenes.random_unit_quats(rng, n)
    t["scale"] = (np.float32(0.8) + np.float32(0.45) * rng.random((n, 3), np.float32)).astype(np.float32)
    return t


def _identity(n):
    t = np.zeros(n, lb.TRANSFORM_DTYPE)
    t["rot"][:, 3] = 1.0
    t["scale"] = 1.0
    return t


def _forest(widths, seed, chains=False):
    """Level l holds widths[l] nodes, each under a random node of level l - 1 (the same position for chains); node ids shuffled."""
    rng = np.random.default_rng(seed)
    start = np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)
    level_parents = np.full(start[-1], -1, np.int64)
    for l in range(1, len(widths)):
        k = np.arange(widths[l])
        level_parents[start[l]:start[l + 1]] = start[l - 1] + (k if chains else rng.integers(0, widths[l - 1], widths[l]))
    n = int(start[-1])
    perm = rng.permutation(n)
    parents = np.full(n, -1, np.int32)
    nonroot = level_parents >= 0
    parents[perm[nonroot]] = perm[level_parents[nonroot]]
    return parents


def reference_level_order(parents):
    """The level order create built on the host, in numpy -> (order, parent_pos, level_start, distinct parents), or raises ValueError with
    create's error text."""
    p = np.asarray(parents, np.int64)
    n = len(p)
    bad = np.nonzero(p >= n)[0]
    if len(bad):
        raise ValueError(f"parent index {int(p[bad[-1]])} out of range")
    key = np.where(p < 0, n, p)
    by_parent = np.argsort(key, kind="stable")  # every parent's children ascending; the roots last
    first = np.searchsorted(key[by_parent], np.arange(n + 1), side="left")
    count = np.searchsorted(key[by_parent], np.arange(n + 1), side="right") - first
    level = by_parent[first[n]:first[n] + count[n]]
    order, parent_pos, level_start = [level], [np.full(len(level), -1, np.int64)], [0]
    base, distinct = 0, 0
    while len(level):
        level_start.append(base + len(level))
        c = count[level]
        distinct += int((c > 0).sum())
        total = int(c.sum())
        excl = np.cumsum(c) - c
        idx = np.repeat(first[level] - excl, c) + np.arange(total)
        nxt = by_parent[idx]
        order.append(nxt)
        parent_pos.append(np.repeat(base + np.arange(len(level)), c))
        base += len(level)
        level = nxt
    order = np.concatenate(order)
    if len(order) != n:
        raise ValueError(f"hierarchy has a cycle ({len(order)} of {n} nodes reachable from roots)")
    return order.astype(np.uint32), np.concatenate(parent_pos).astype(np.int32), np.asarray(level_start, np.uint32), distinct


def _expected_bytes(parents, level_start, distinct):
    return (len(parents) - int(level_start[1])) * (52 + 4 + 52) + distinct * 52


def _assert_layout(h, parents, what):
    order, parent_pos, level_start, distinct = reference_level_order(parents)
    got = h.levelOrder()
    assert h.n == len(parents)
    assert h.depth == len(level_start) - 1, f"{what}: depth"
    assert np.array_equal(got[0], order), f"{what}: level order"
    assert np.array_equal(got[1], parent_pos), f"{what}: parent positions"
    assert np.array_equal(got[2], level_start), f"{what}: level starts"
    assert h.algorithmic_bytes() == _expected_bytes(parents, level_start, distinct), f"{what}: algorithmic bytes"


def _set_parents(ctx, h, parents, entry, max_blocks):
    if entry == "host":
        h.setParents(parents)
        return
    p = np.ascontiguousarray(parents, np.int32)
    d = ctx.to_device(p)
    try:
        h.setParentsDevice(d, len(p), max_blocks=max_blocks)
    finally:
        ctx.free_device(d)


def _star(n_children):
    return np.concatenate([[-1], np.zeros(n_children, np.int32)]).astype(np.int32)


SHAPES = {
    **{f"chain_{d}": (lambda d=d: _forest([40] * d, seed=d, chains=True)) for d in (1, 2, 30, 31, 32, 33, 300)},
    "8192_then_8193": lambda: _forest([5, 8192, 8193, 40], seed=8),
    "8193_first": lambda: _forest([1, 8193, 8192, 3], seed=9),
    "narrow_wide_narrow_wide": lambda: _forest([3, 100, 20000, 7, 9000, 5], seed=10),
    "odd_widths": lambda: _forest([7, 300, 1000, 2500, 513, 8191], seed=11),
    "single_node": lambda: np.array([-1], np.int32),
    "star_195": lambda: _star(195),
    "roots_only": lambda: np.full(1000, -1, np.int32),
    "parents_below_minus_1": lambda: np.where(_forest([20, 300, 900], seed=12) < 0, np.random.default_rng(1).integers(-1000, -1, 1220), _forest([20, 300, 900], seed=12)).astype(np.int32),
    "config3_1m": lambda: scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)[0],
}


@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_same_layout_as_reference_bfs(ctx, shape, entry):
    """create(A) then set_parents(B) holds what create(B) holds and what the numpy BFS of B gives: level order, parent positions, level
    starts, depth and algorithmic bytes.  The device entry at max_blocks 1, 2, 3 and the default; the host entry (an upload in front of the
    same builder) at the default grid."""
    b = SHAPES[shape]()
    a = _forest([3, 17, 60], seed=len(b))  # another size and shape: every set_parents below changes n
    fresh = lb.Hierarchy(ctx, b)
    _assert_layout(fresh, b, f"{shape}: create")
    fresh_layout = fresh.levelOrder()
    h = lb.Hierarchy(ctx, a)
    for mb in (GRIDS if entry == "device" else (0,)):
        what = f"{shape}, {entry} entry, max_blocks {mb}"
        _set_parents(ctx, h, b, entry, mb)
        _assert_layout(h, b, what)
        for x, y in zip(h.levelOrder(), fresh_layout):
            assert np.array_equal(x, y), f"{what}: differs from create"
        assert h.algorithmic_bytes() == fresh.algorithmic_bytes() and h.depth == fresh.depth
        _set_parents(ctx, h, a, entry, mb)
        _assert_layout(h, a, f"{what}, back to A")
    h.close()
    fresh.close()


class _Tracked:
    """A hierarchy with the locals and globals it must hold, per node index; propagate is checked against the oracle."""

    def __init__(self, ctx, oracle, parents, seed):
        rng = np.random.default_rng(seed)
        self.ctx, self.oracle, self.rng = ctx, oracle, rng
        self.parents = parents.copy()
        n = len(parents)
        self.locals = _transforms(rng, n, (10.0, 10.0, 10.0))
        roots = _transforms(rng, n, (6000.0, 300.0, 6000.0))
        self.h = lb.Hierarchy(ctx, parents)
        self.h.setLocalTransforms(self.locals)
        self.h.setRootTransforms(roots)
        self.globals = roots.copy()
        self.propagate_and_check("initial")

    def set_parents(self, parents, what, entry="host", max_blocks=0):
        n_old = len(self.parents)
        _set_parents(self.ctx, self.h, parents, entry, max_blocks)
        n = len(parents)
        keep = min(n_old, n)
        locals_, globals_ = _identity(n), _identity(n)
        locals_[:keep] = self.locals[:keep]
        globals_[:keep] = self.globals[:keep]
        self.parents, self.locals, self.globals = parents.copy(), locals_, globals_
        _assert_layout(self.h, parents, what)
        assert_transforms_equal(self.h.getLocalTransforms(), self.locals, f"{what}: locals follow their nodes")
        assert_transforms_equal(self.h.getTransforms(), self.globals, f"{what}: globals follow their nodes")

    def set_subset(self, nodes, values, globals_=False):
        self.h.setSubset(nodes, values, globals_=globals_)
        (self.globals if globals_ else self.locals)[np.asarray(nodes)] = values

    def propagate_and_check(self, what, radii=True):
        self.h.propagate()
        exp = self.oracle.propagate(self.parents, _as_bytes(self.locals), _as_bytes(self.globals)).view(lb.TRANSFORM_DTYPE).reshape(-1)
        assert_transforms_equal(self.h.getTransforms(), exp, f"{what}: propagated globals")
        self.globals = exp.copy()
        n = len(self.parents)
        br = np.linspace(0.25, 4.0, n).astype(np.float32)
        pos, rad = self.h.getSpheres(br)
        assert_bits_equal(pos, exp["pos"], f"{what}: sphere positions")
        assert_bits_equal(rad, self.oracle.sphere_radius(_as_bytes(exp), br), f"{what}: sphere radii")
        base = (1500.25, -80.0, 3000.5)
        assert_bits_equal(self.h.getRelativeMatrices(base), self.oracle.relative_matrices(_as_bytes(exp), base), f"{what}: relative matrices")
        return exp


def _subtree(parents, x):
    """x and every node below it."""
    inside = np.zeros(len(parents), bool)
    inside[x] = True
    while True:
        grow = (parents >= 0) & ~inside
        grow[grow] = inside[parents[grow]]
        if not grow.any():
            return inside
        inside |= grow


def _depths(parents):
    order, _, level_start, _ = reference_level_order(parents)
    d = np.zeros(len(parents), np.int64)
    for l in range(len(level_start) - 1):
        d[order[level_start[l]:level_start[l + 1] if l + 1 < len(level_start) else len(parents)]] = l
    return d


@pytest.mark.parametrize("entry,max_blocks", [("host", 0), ("device", 0), ("device", 2)])
def test_transforms_follow_their_nodes(ctx, oracle, entry, max_blocks):
    """Subtrees moved deeper and shallower, a node detached to a root, a root attached under a leaf, a World-style swap-remove, and a setSubset
    queued right before the call: the locals and globals of every surviving node are where its index says, and propagate, spheres and
    relative matrices equal the oracle on the new parents."""
    t = _Tracked(ctx, oracle, _forest([5, 40, 200, 800, 1500], seed=21), seed=22)
    rng = np.random.default_rng(23)

    def edit(parents, what):
        t.set_parents(parents, what, entry, max_blocks)
        t.propagate_and_check(what)

    p = t.parents.copy()
    d = _depths(p)
    x = int(rng.choice(np.nonzero(d == 1)[0]))  # deeper: a level-1 subtree under a level-3 node of another tree
    target = int(rng.choice(np.nonzero((d == 3) & ~_subtree(p, x))[0]))
    p[x] = target
    edit(p, "subtree moved deeper")

    p = t.parents.copy()
    d = _depths(p)
    x = int(rng.choice(np.nonzero(d >= 4)[0]))  # shallower: a deep node under a root
    p[x] = int(rng.choice(np.nonzero(p < 0)[0]))
    edit(p, "subtree moved shallower")

    p = t.parents.copy()
    x = int(rng.choice(np.nonzero(p >= 0)[0]))  # detached: its global (kept) is now its root transform
    p[x] = -1
    edit(p, "node detached to a root")

    p = t.parents.copy()
    r = int(rng.choice(np.nonzero(p < 0)[0]))  # a root attached under a leaf of another tree: its local (kept) now composes
    has_child = np.zeros(len(p), bool)
    has_child[p[p >= 0]] = True
    leaf = int(rng.choice(np.nonzero(~has_child & ~_subtree(p, r))[0]))
    p[r] = leaf
    edit(p, "root attached under a leaf")

    # World::destroyEntity of a hierarchy node (world.cpp:633-637): the last node takes the freed index, n shrinks by one; its transforms are
    # moved to that index by the caller (the library keeps the removed node's there)
    p = t.parents.copy()
    n = len(p)
    has_child = np.zeros(n, bool)
    has_child[p[p >= 0]] = True
    v = int(rng.choice(np.nonzero(~has_child[:-1] & (p[:-1] != n - 1))[0]))
    last_local, last_global, last_is_root = t.locals[n - 1].copy(), t.globals[n - 1].copy(), p[n - 1] < 0
    p[v] = p[n - 1]
    p[p == n - 1] = v
    p = p[:-1].copy()
    t.set_parents(p, "swap-remove", entry, max_blocks)
    t.set_subset([v], last_local[None])
    if last_is_root:
        t.set_subset([v], last_global[None], globals_=True)
    t.propagate_and_check("swap-remove")

    # a setSubset queued right before the call lands in the values the new topology carries
    nodes = rng.choice(len(t.parents), 300, replace=False).astype(np.uint32)
    t.set_subset(nodes, _transforms(rng, len(nodes), (10.0, 10.0, 10.0)))
    roots = np.nonzero(t.parents < 0)[0][:3].astype(np.uint32)
    t.set_subset(roots, _transforms(rng, len(roots), (6000.0, 300.0, 6000.0)), globals_=True)
    p = t.parents.copy()
    x = int(rng.choice(np.nonzero(p >= 0)[0]))
    p[x] = -1
    edit(p, "setSubset queued before the call")
    t.h.close()


def test_grow_and_shrink(ctx, oracle):
    """n + 1, n + 10 000 (new nodes read back as the identity, under old and new parents), then shrinks; refreshSpheres without radii is
    refused after a size change and equals the oracle with them."""
    t = _Tracked(ctx, oracle, _forest([10, 90, 700, 3000], seed=31), seed=32)
    rng = np.random.default_rng(33)
    br0 = (np.float32(0.5) + rng.random(len(t.parents), np.float32)).astype(np.float32)
    t.h.refreshSpheres(br0)
    t.h.refreshSpheres(None)  # the same n: the radii are kept

    def grow(k, what):
        n = len(t.parents)
        extra = np.empty(k, np.int32)
        for j in range(k):  # under an old node or under one of the new ones before it
            extra[j] = rng.integers(0, n + j)
        t.set_parents(np.concatenate([t.parents, extra]), what)
        assert_transforms_equal(t.h.getLocalTransforms()[n:], _identity(k), f"{what}: new locals are the identity")
        assert_transforms_equal(t.h.getTransforms()[n:], _identity(k), f"{what}: new globals are the identity")
        t.set_subset(np.arange(n, n + k, dtype=np.uint32), _transforms(rng, k, (10.0, 10.0, 10.0)))

    def spheres(what):
        with pytest.raises(lb.LumixB200Error) as e:
            t.h.refreshSpheres(None)
        assert e.value.code == _lib.ERR_INVALID
        exp = t.propagate_and_check(what)
        n = len(t.parents)
        br = (np.float32(0.5) + rng.random(n, np.float32)).astype(np.float32)
        d_pos, d_rad = t.h.refreshSpheres(br)
        assert_bits_equal(ctx.copy_to_host(d_pos, 3 * n, np.float64).reshape(n, 3), exp["pos"], f"{what}: refreshed sphere positions")
        assert_bits_equal(ctx.copy_to_host(d_rad, n, np.float32), oracle.sphere_radius(_as_bytes(exp), br), f"{what}: refreshed sphere radii")

    grow(1, "grow by 1")
    spheres("grow by 1")
    grow(10_000, "grow by 10 000")
    spheres("grow by 10 000")
    # shrink below the original size: nodes whose parent leaves become roots
    m = len(t.parents) - 12_000
    p = t.parents[:m].copy()
    p[p >= m] = -1
    t.set_parents(p, "shrink by 12 000")
    spheres("shrink by 12 000")
    t.h.close()


def test_config3_chain_after_reparent(ctx, oracle):
    """Config 3 (1 M nodes): propagate -> refreshSpheres -> CullingSystem.set_many_device -> cull, then a subtree re-parented on the device
    and the chain again: the visible set equals the oracle's on the new parents."""
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    n = len(parents)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    bounding = np.full(n, 1.0, np.float32)
    pos0, rad0 = h.getSpheres(bounding)
    cs = lb.CullingSystem(ctx)
    cs.add(np.arange(n, dtype=np.int32), np.zeros(n, np.uint8), pos0, rad0)
    cs.flush()
    f = lb.frustum_perspective(**scenes.c2_frustum_args())
    rng = np.random.default_rng(41)
    root_ids = np.nonzero(parents < 0)[0]
    p = parents.copy()
    for _ in range(3):  # three subtrees, each from one tree to a node of another
        x = int(rng.choice(np.nonzero(p >= 0)[0]))
        target = int(rng.choice(root_ids))
        while _subtree(p, x)[target]:
            target = int(rng.choice(root_ids))
        p[x] = target
    d = ctx.to_device(p)
    h.setParentsDevice(d, n)
    ctx.free_device(d)
    h.propagate()
    d_pos, d_rad = h.refreshSpheres(None)  # n unchanged: the radii are kept
    cs.set_many_device(d_pos, d_rad, n)
    got = np.sort(cs.cull(f).ids)
    exp = oracle.propagate(p, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    oc = oracle.OracleCulling()
    oc.add(np.arange(n, dtype=np.int32), np.zeros(n, np.uint8), exp["pos"], oracle.sphere_radius(_as_bytes(exp), bounding))
    oids, _, _ = oc.cull(lb.culling.frustum_bytes(f))
    assert len(oids) > 1000
    assert np.array_equal(got, np.sort(oids)), "visible set after the re-parent differs from the oracle"
    cs.close()
    h.close()


def _cycle_cases():
    base = _forest([4, 30, 200], seed=51)
    n = len(base)
    self_parent = base.copy()
    self_parent[17] = 17
    two = base.copy()
    two[5], two[9] = 9, 5
    loop = np.concatenate([base, n + (np.arange(50) + 1) % 50]).astype(np.int32)  # a 50-node loop beside the valid forest
    equal_n = base.copy()
    equal_n[40] = n
    two_bad = base.copy()
    two_bad[3], two_bad[100] = n + 7, n + 2  # create names the parent of the highest offending node
    return {"self_parent": self_parent, "two_cycle": two, "loop_50": loop, "parent_equals_n": equal_n, "two_out_of_range": two_bad}


@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("case", list(_cycle_cases()))
def test_refusal_leaves_the_hierarchy_as_it_was(ctx, oracle, case, entry):
    bad = _cycle_cases()[case]
    with pytest.raises(ValueError) as ref:
        reference_level_order(bad)
    with pytest.raises(lb.LumixB200Error) as e:
        lb.Hierarchy(ctx, bad)
    assert e.value.code == _lib.ERR_INVALID and str(ref.value) in str(e.value), "create's refusal"
    valid = bad.copy()  # the same n, the offending entries made roots: the refused call is the only difference
    valid[(valid >= len(valid)) | (np.arange(len(valid)) == valid)] = -1
    if case == "two_cycle":
        valid[5] = -1
    elif case == "loop_50":
        valid[-50] = -1
    reference_level_order(valid)
    t = _Tracked(ctx, oracle, valid, seed=53)
    before = t.h.levelOrder(), t.h.depth, t.h.getLocalTransforms(), t.h.getTransforms()
    for mb in (GRIDS if entry == "device" else (0,)):
        with pytest.raises(lb.LumixB200Error) as e:
            _set_parents(ctx, t.h, bad, entry, mb)
        assert e.value.code == _lib.ERR_INVALID and str(ref.value) in str(e.value), f"max_blocks {mb}: refusal text"
        assert t.h.n == len(t.parents) and t.h.depth == before[1]
        for x, y in zip(t.h.levelOrder(), before[0]):
            assert np.array_equal(x, y), "the level order changed on a refusal"
        assert_transforms_equal(t.h.getLocalTransforms(), before[2], "locals after a refusal")
        assert_transforms_equal(t.h.getTransforms(), before[3], "globals after a refusal")
        t.propagate_and_check(f"{case}, max_blocks {mb}: propagate after a refusal")
    t.h.close()


def test_n_zero_is_refused(ctx):
    h = lb.Hierarchy(ctx, _forest([3, 10], seed=61))
    before = h.levelOrder()
    L = _lib.lib()
    empty = np.zeros(1, np.int32)
    assert L.lb200_hierarchy_set_parents(h.h, _lib.ptr(empty), C.c_uint32(0)) == _lib.ERR_INVALID
    d = ctx.to_device(empty)
    assert L.lb200_hierarchy_set_parents_device(h.h, C.c_void_p(d), C.c_uint32(0), C.c_uint32(0)) == _lib.ERR_INVALID
    ctx.free_device(d)
    assert h.n == 13 and h.depth == 2
    for x, y in zip(h.levelOrder(), before):
        assert np.array_equal(x, y)
    h.close()


def test_launch_count_does_not_grow_with_depth(ctx):
    """A depth-300 chain and a depth-2 forest: the same number of launches per set_parents, from either entry point."""
    chain = _forest([40] * 300, seed=71, chains=True)
    flat = _forest([100, 11900], seed=72)
    deltas = []
    for parents in (chain, flat):
        h = lb.Hierarchy(ctx, parents)
        d = ctx.to_device(parents)
        ctx.synchronize()
        before = ctx.launches
        h.setParents(parents)
        host = ctx.launches - before
        before = ctx.launches
        h.setParentsDevice(d, len(parents))
        dev = ctx.launches - before
        ctx.free_device(d)
        deltas.append((host, dev))
        h.close()
    assert deltas[0] == deltas[1], f"launches per set_parents: depth 300 {deltas[0]}, depth 2 {deltas[1]}"
    assert deltas[0][0] == deltas[0][1]


SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libengine_shim_b200.so")


def test_world_patch_reparents_every_round(oracle):
    """host/world_b200.inl inside the reference's own World, re-parenting between each of 5 rounds at 60 k entities: propagateHierarchyB200
    re-parents its hierarchy on the device and must leave the transforms and `transformed` counts of the reference recursion."""
    if not os.path.exists(SO):
        pytest.skip("oracle/_ref/libengine_shim_b200.so not built (needs the reference sources at build time)")
    shim = C.CDLL(SO)
    os.environ["LB200_ENGINE_SHIM_LOADED"] = "1"  # the engine's job system cannot be shut down on Linux: tests/conftest.py leaves with os._exit
    n, rounds = 60_000, 5
    parents, locals_, roots = scenes.hierarchy_forest(n, 8, 4, seed=29)
    rng = np.random.default_rng(6)
    listens = (rng.random(n) < 0.7).astype(np.uint8)
    root_ids = np.nonzero(parents < 0)[0].astype(np.uint32)
    moved = rng.choice(root_ids, max(1, len(root_ids) // 2), replace=False).astype(np.uint32)
    vals = np.zeros((rounds, len(moved)), lb.TRANSFORM_DTYPE)
    for r in range(rounds):
        vals[r]["pos"] = roots[moved]["pos"] + rng.normal(size=(len(moved), 3)) * 50.0
        vals[r]["rot"] = scenes.random_unit_quats(rng, len(moved))
        vals[r]["scale"] = (0.7 + 0.6 * rng.random((len(moved), 3))).astype(np.float32)
    out_ref, out_b = np.zeros(n, lb.TRANSFORM_DTYPE), np.zeros(n, lb.TRANSFORM_DTYPE)
    calls_ref, calls_b = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    seconds = np.zeros(2)
    world_locals = np.zeros(n, lb.TRANSFORM_DTYPE)
    p_ = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    shim.wshim_run.restype = C.c_int
    rc = shim.wshim_run(p_(parents), p_(np.ascontiguousarray(locals_)), p_(np.ascontiguousarray(roots)), C.c_uint32(n), p_(listens),
                        p_(moved), p_(np.ascontiguousarray(vals)), C.c_uint32(len(moved)), C.c_uint32(rounds), C.c_int(1),
                        p_(out_ref), p_(out_b), p_(calls_ref), p_(calls_b), p_(seconds), p_(world_locals))
    assert rc == 0
    for field in ("pos", "rot", "scale"):
        assert out_ref[field].tobytes() == out_b[field].tobytes(), "World::propagateHierarchyB200 left other transforms than World::transformEntity"
    assert np.array_equal(calls_ref, calls_b), "the `transformed` delegates fired for other entities than under the reference recursion"
    assert calls_ref.sum() > 0 and (calls_ref[listens == 0] == 0).all()
