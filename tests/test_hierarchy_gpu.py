"""GPU parity of the batched hierarchy propagation against the oracle's transformEntity restatement.

The kernels keep the reference's op order (fp64 position, no FMA), so propagated globals, computed locals and relative
matrices must equal the oracle's bit for bit (DESIGN §2); north_star's 1e-5 relative tolerance is not what these tests allow.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from bitexact import assert_bits_equal, assert_transforms_equal

pytestmark = pytest.mark.gpu


def _as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)


def _check(got, exp):
    assert_transforms_equal(got, exp, "propagated globals")
    return True


@pytest.mark.parametrize("n,depth,fanout", [(20_000, 8, 3), (5000, 3, 7), (1000, 1, 2), (50_000, 12, 2)])
def test_forest_matches_oracle(ctx, oracle, n, depth, fanout):
    parents, locals_, roots = scenes.hierarchy_forest(n, depth, fanout, seed=n)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    got = h.getTransforms()
    exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    _check(got, exp)  # visibility after a re-cull needs exact positions
    # sphere refresh (render_module.cpp:1544-1554)
    br = np.linspace(0.5, 3.0, len(parents)).astype(np.float32)
    pos, rad = h.getSpheres(br)
    assert np.array_equal(pos, exp["pos"])
    assert np.array_equal(rad, oracle.sphere_radius(_as_bytes(exp), br))


def test_shuffled_node_order(ctx, oracle):
    """Nodes arrive in arbitrary order (children before parents): the level sort must not change results."""
    parents, locals_, roots = scenes.hierarchy_forest(30_000, 6, 4, seed=77)
    rng = np.random.default_rng(5)
    perm = rng.permutation(len(parents))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    p2 = np.where(parents[perm] >= 0, inv[np.maximum(parents[perm], 0)], -1).astype(np.int32)
    h = lb.Hierarchy(ctx, p2)
    h.setLocalTransforms(locals_[perm])
    h.setRootTransforms(roots[perm])
    h.propagate()
    got = h.getTransforms()
    exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    assert _check(got, exp[perm])


def test_propagate_then_cull(ctx, oracle):
    """Config 3 end to end: propagate -> sphere refresh -> CullingSystem::set -> cull; visibility bit-exact."""
    parents, locals_, roots = scenes.hierarchy_forest(100_000, 6, 5, seed=9, root_extent=(2000.0, 200.0, 2000.0))
    n = len(parents)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    br = np.full(n, 1.0, np.float32)
    pos, rad = h.getSpheres(br)
    ent = np.arange(n, dtype=np.int32)
    cs = lb.CullingSystem(ctx)
    # entities start somewhere else, then move (onModelInstanceMoved -> CullingSystem::set)
    cs.add(ent, np.zeros(n, np.uint8), np.zeros((n, 3)), br)
    cs.set(ent, pos, rad)
    exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    oc = oracle.OracleCulling()
    oc.add(ent, np.zeros(n, np.uint8), np.zeros((n, 3)), br)
    oc.set(ent, exp["pos"], oracle.sphere_radius(_as_bytes(exp), br))
    f = lb.frustum_perspective(**scenes.c1_frustum_args())
    res = cs.cull(f)
    oids, _, _ = oc.cull(lb.culling.frustum_bytes(f))
    assert np.array_equal(np.sort(res.ids), np.sort(oids))


def test_1m_depth8_properties(ctx):
    """Full C3 size: identity locals reproduce the root transform in every descendant; re-running is idempotent."""
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    h = lb.Hierarchy(ctx, parents)
    assert h.depth == 8
    ident = np.zeros(len(parents), lb.TRANSFORM_DTYPE)
    ident["rot"][:, 3] = 1.0
    ident["scale"] = 1.0
    roots2 = roots.copy()
    roots2["rot"] = 0.0
    roots2["rot"][:, 3] = 1.0
    roots2["scale"] = 1.0
    h.setLocalTransforms(ident)
    h.setRootTransforms(roots2)
    h.propagate()
    g = h.getTransforms()
    root_of = np.arange(len(parents))
    for _ in range(8):
        root_of = np.where(parents[root_of] >= 0, parents[root_of], root_of)
    assert np.array_equal(g["pos"], roots2["pos"][root_of])
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    a = h.getTransforms()
    h.propagate()
    b = h.getTransforms()
    assert np.array_equal(_as_bytes(a)[:, :52], _as_bytes(b)[:, :52])
    assert np.all(np.isfinite(a["pos"]))


def test_relative_matrices_match_oracle(ctx, oracle):
    """World::getRelativeMatrix of every propagated node against a camera position (world.cpp:370-377), bit for bit."""
    parents, locals_, roots = scenes.hierarchy_forest(30_000, 6, 4, seed=77)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    globals_ = h.getTransforms()
    for base in ((0.0, 0.0, 0.0), (1500.25, -80.0, 3000.5), (-5999.0, 299.0, 5999.0)):
        got = h.getRelativeMatrices(base)
        exp = oracle.relative_matrices(_as_bytes(globals_), base)
        assert_bits_equal(got, exp, f"relative matrices against {base}")
    h.close()


def test_compute_locals_match_oracle(ctx, oracle):
    """World::transformEntity(update_local) batched: locals from authoritative globals (Transform::computeLocal, math.cpp:809-816),
    bit for bit against the oracle; then propagate brings the globals back within the 1e-5 relative tolerance of north_star (a round
    trip through computeLocal and compose is not exact in the reference either)."""
    parents, locals_, roots = scenes.hierarchy_forest(40_000, 7, 3, seed=5)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    globals_ = h.getTransforms()
    # move every node in world space (as physics would), then ask for the locals that reproduce it
    rng = np.random.default_rng(9)
    moved = globals_.copy()
    moved["pos"] += rng.normal(size=moved["pos"].shape) * 3.0
    h.setTransforms(moved)
    h.computeLocalTransforms()
    got = h.getLocalTransforms()
    exp = oracle.compute_locals(parents, _as_bytes(moved), _as_bytes(locals_)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    nonroot = parents >= 0
    assert nonroot.sum() > 30_000
    assert_transforms_equal(got, exp, "computed locals", rows=nonroot)
    # round trip: propagate with the new locals reproduces the moved world transforms
    h.propagate()
    back = h.getTransforms()
    err = np.abs(back["pos"] - moved["pos"]).max()
    assert err < 1e-5 * max(1.0, np.abs(moved["pos"]).max()), err
    h.close()


def test_c3_1m_equals_oracle_at_full_size(ctx, oracle):
    """BASELINE configs[2] at its stated size: the 1 M-node, depth-8 forest propagated on the GPU against the C restatement of
    World::transformEntity (serial DFS, ~35 ms), every Transform bit for bit, and the sphere refresh behind it."""
    parents, locals_, roots = scenes.hierarchy_forest(1_000_000, 8, 7, seed=3)
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    got = h.getTransforms()
    exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    for field in ("pos", "rot", "scale"):
        assert got[field].tobytes() == exp[field].tobytes(), f"1 M-node propagate: {field} differs from the oracle"
    br = np.full(len(parents), 1.0, np.float32)
    pos, rad = h.getSpheres(br)
    assert pos.tobytes() == np.ascontiguousarray(exp["pos"]).tobytes()
    assert np.array_equal(rad, oracle.sphere_radius(_as_bytes(exp), br))
    h.close()
