"""Bit-for-bit comparison of kernel outputs with the oracle (DESIGN §2: pose, palettes, skinned vertices, propagated, local and
relative transforms are bit-exact).  Shared by the GPU test modules; the failure message names the first element that differs."""
import numpy as np

_UINT = {2: np.uint16, 4: np.uint32, 8: np.uint64}


def assert_bits_equal(got, exp, what):
    """got and exp hold the same bit patterns (so -0.0 != 0.0, and NaNs compare by payload)."""
    g, e = np.ascontiguousarray(got), np.ascontiguousarray(exp)
    assert g.shape == e.shape and g.dtype == e.dtype, f"{what}: {g.dtype}{g.shape} against {e.dtype}{e.shape}"
    gb, eb = g.view(_UINT[g.dtype.itemsize]), e.view(_UINT[e.dtype.itemsize])
    diff = gb != eb
    if diff.any():
        first = tuple(int(i) for i in np.argwhere(diff)[0])
        err = np.abs(g.astype(np.float64) - e.astype(np.float64))
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.size} values differ in their bits; first at {first}: "
                             f"{g[first]!r} against {e[first]!r}; largest abs difference {np.nanmax(err)}")


def assert_transforms_equal(got, exp, what, rows=None):
    """Engine Transforms (TRANSFORM_DTYPE): pos, rot and scale bit for bit, on `rows` (a mask or index array) or all of them."""
    for field in ("pos", "rot", "scale"):
        g, e = got[field], exp[field]
        if rows is not None:
            g, e = g[rows], e[rows]
        assert_bits_equal(g, e, f"{what}: {field}")
