"""The hierarchy kernels at the edges of their launch plan, bit for bit against the oracle.

lb200_hierarchy_propagate runs the leading levels of at most SMALL_LEVEL_NODES = 8192 nodes in one block (at most MAX_SMALL_LEVELS = 30
of them), then one launch per level chained by programmatic dependent launch.  The shapes here cross each of those switches: depths
around 31 / 32 levels, levels of exactly 8192 and 8193 nodes, a wide first level, narrow levels after wide ones and widths that are
not multiples of the 256-thread block.  setSubset (double-buffered pinned staging that grows on demand) and refreshSpheres are the
per-frame entry points of config 3.
"""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes
from bitexact import assert_bits_equal, assert_transforms_equal

pytestmark = pytest.mark.gpu


def _as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)


def _transforms(rng, n, extent):
    t = np.zeros(n, lb.TRANSFORM_DTYPE)
    t["pos"] = (rng.random((n, 3)) * 2.0 - 1.0) * np.asarray(extent, np.float64)
    t["rot"] = scenes.random_unit_quats(rng, n)
    t["scale"] = (np.float32(0.8) + np.float32(0.45) * rng.random((n, 3), np.float32)).astype(np.float32)  # never 0: computeLocal divides by it
    return t


def _forest(widths, seed, chains=False):
    """Level l holds widths[l] nodes; each picks a random parent on level l - 1 (or the same position, for chains).  Node ids are
    shuffled so parents and children come in any order.  -> parents i32[n], locals, root globals."""
    rng = np.random.default_rng(seed)
    start = np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)
    level_parents = np.full(start[-1], -1, np.int64)
    for l in range(1, len(widths)):
        k = np.arange(widths[l])
        level_parents[start[l]:start[l + 1]] = start[l - 1] + (k if chains else rng.integers(0, widths[l - 1], widths[l]))
    n = int(start[-1])
    perm = rng.permutation(n)  # level-order node k becomes node perm[k]
    parents = np.full(n, -1, np.int32)
    nonroot = level_parents >= 0
    parents[perm[nonroot]] = perm[level_parents[nonroot]]
    return parents, _transforms(rng, n, (10.0, 10.0, 10.0)), _transforms(rng, n, (6000.0, 300.0, 6000.0))


def _check_all(ctx, oracle, parents, locals_, roots, what):
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    exp = oracle.propagate(parents, _as_bytes(locals_), _as_bytes(roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    assert_transforms_equal(h.getTransforms(), exp, f"{what}: propagated globals")
    br = np.linspace(0.25, 4.0, len(parents)).astype(np.float32)
    pos, rad = h.getSpheres(br)
    assert_bits_equal(pos, exp["pos"], f"{what}: sphere positions")
    assert_bits_equal(rad, oracle.sphere_radius(_as_bytes(exp), br), f"{what}: sphere radii")
    for base in ((0.0, 0.0, 0.0), (1500.25, -80.0, 3000.5)):
        assert_bits_equal(h.getRelativeMatrices(base), oracle.relative_matrices(_as_bytes(exp), base), f"{what}: relative matrices against {base}")
    # world transforms authoritative: move every node, then derive the locals (roots keep the locals uploaded above)
    rng = np.random.default_rng(len(parents))
    moved = exp.copy()
    moved["pos"] += rng.normal(size=moved["pos"].shape) * 3.0
    h.setTransforms(moved)
    h.computeLocalTransforms()
    exp_locals = oracle.compute_locals(parents, _as_bytes(moved), _as_bytes(locals_)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    assert_transforms_equal(h.getLocalTransforms(), exp_locals, f"{what}: computed locals")
    return h


@pytest.mark.parametrize("depth", [1, 2, 30, 31, 32, 33, 300])
def test_chain_depths(ctx, oracle, depth):
    """31 levels are the most one small-levels launch takes (30 below the roots); 32 adds the first per-level launch."""
    parents, locals_, roots = _forest([40] * depth, seed=depth, chains=True)
    h = _check_all(ctx, oracle, parents, locals_, roots, f"depth {depth}")
    assert h.depth == depth
    h.close()


WIDTHS = {
    "8192_then_8193": [5, 8192, 8193, 40],         # 8192 stays in the small-levels block, 8193 and the narrow level after it do not
    "8193_first": [1, 8193, 8192, 3],              # no small-levels launch at all
    "narrow_wide_narrow_wide": [3, 100, 20000, 7, 9000, 5],
    "odd_widths": [7, 300, 1000, 2500, 513, 8191],  # all in one small-levels launch, none a multiple of 256
}


@pytest.mark.parametrize("shape", list(WIDTHS))
def test_level_widths(ctx, oracle, shape):
    widths = WIDTHS[shape]
    parents, locals_, roots = _forest(widths, seed=len(widths) * 1000 + widths[1])
    h = _check_all(ctx, oracle, parents, locals_, roots, shape)
    assert h.depth == len(widths)
    h.close()


def test_set_subset_back_to_back_then_refresh_spheres(ctx, oracle):
    """setSubset calls queued without a read in between (roots and locals; 0, 1, 100 and 5000 nodes, the last growing the staging
    mid-sequence; nodes repeated in later calls, whose values must win), then propagate and refreshSpheres, read through the device
    pointers it returns; a second round reuses the stored radii."""
    widths = [150, 400, 3000, 9000]
    parents, locals_, roots = _forest(widths, seed=8)
    n = len(parents)
    root_ids = np.nonzero(parents < 0)[0]
    child_ids = np.nonzero(parents >= 0)[0]
    h = lb.Hierarchy(ctx, parents)
    h.setLocalTransforms(locals_)
    h.setRootTransforms(roots)
    h.propagate()
    rng = np.random.default_rng(3)
    exp_locals, exp_roots = locals_.copy(), roots.copy()

    def edit(ids, globals_):
        ids = np.asarray(ids, np.uint32)
        values = _transforms(rng, len(ids), (6000.0, 300.0, 6000.0) if globals_ else (10.0, 10.0, 10.0))
        h.setSubset(ids, values, globals_=globals_)
        (exp_roots if globals_ else exp_locals)[ids] = values
        values["pos"] = np.nan  # the library copied them: later changes to the caller's array must not reach the device
        ids[:] = 0

    first_roots = rng.choice(root_ids, 100, replace=False)
    first_children = rng.choice(child_ids, 100, replace=False)
    edit([], True)
    edit(first_roots[:1], True)
    edit([], False)
    edit(first_children[:1], False)
    edit(first_roots, True)
    edit(first_children, False)
    edit(rng.choice(child_ids, 5000, replace=False), False)  # grows the staging while earlier uploads may be in flight
    edit(first_children[::7], False)  # repeated nodes: this later value wins
    edit(first_roots[:1], True)
    edit(first_roots[::3], True)
    h.propagate()
    exp = oracle.propagate(parents, _as_bytes(exp_locals), _as_bytes(exp_roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    br = (np.float32(0.5) + rng.random(n, np.float32)).astype(np.float32)
    dev_pos, dev_rad = h.refreshSpheres(br)
    assert_bits_equal(ctx.copy_to_host(dev_pos, 3 * n, np.float64).reshape(n, 3), exp["pos"], "refreshed sphere positions")
    assert_bits_equal(ctx.copy_to_host(dev_rad, n, np.float32), oracle.sphere_radius(_as_bytes(exp), br), "refreshed sphere radii")
    assert_transforms_equal(h.getTransforms(), exp, "globals after the subset edits")

    # second round: more edits, propagate, refresh with the radii kept from the first call
    edit(rng.choice(root_ids, 37, replace=False), True)
    edit(rng.choice(child_ids, 250, replace=False), False)
    h.propagate()
    exp = oracle.propagate(parents, _as_bytes(exp_locals), _as_bytes(exp_roots)).view(lb.TRANSFORM_DTYPE).reshape(-1)
    dev_pos2, dev_rad2 = h.refreshSpheres(None)
    assert (dev_pos2, dev_rad2) == (dev_pos, dev_rad)
    assert_bits_equal(ctx.copy_to_host(dev_pos2, 3 * n, np.float64).reshape(n, 3), exp["pos"], "second refresh: sphere positions")
    assert_bits_equal(ctx.copy_to_host(dev_rad2, n, np.float32), oracle.sphere_radius(_as_bytes(exp), br), "second refresh: sphere radii")
    h.close()
