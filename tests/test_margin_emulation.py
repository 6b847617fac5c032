"""CPU emulation (numpy float32, no FMA) of the two conservative shortcuts of the cull kernels, checked against the exact expressions:

* plane masking (plane_mask over relative_offsets, csrc/cull_common.cuh): a plane dropped for a cell can never give a sphere of that
  cell a negative t - r (test_rows);
* the cheap pass A1 (outside_by_margin, csrc/cull_common.cuh): a page it drops is classified "outside" by the exact cell tests of
  classify_cell (neither containsAABB(origin + cs, cs) nor intersectsAABB(origin - cs, 2cs), geometry.cpp:99-118, 159-178).

Both cull kernels call these functions.  The emulation repeats their expressions operation by operation; frustums come from the
product's own host builders."""
import numpy as np

import lumixengine_b200 as lb
from lumixengine_b200 import culling

F = np.float32
CS = F(300.0)
POINT_OF_PLANE = [0, 4, 1, 0, 0, 2]  # geometry.cpp:134-142, planes NEAR FAR LEFT RIGHT TOP BOTTOM


def _planes(f):
    xs, ys, zs, ds = (np.array(getattr(f, k)[:], F) for k in ("xs", "ys", "zs", "ds"))
    pts = np.array([list(p) for p in f.points], F)
    # the kernels use the 6 distinct planes: indices 2..7 of the 8-plane arrays (EXTRA0/1 duplicate NEAR)
    return xs[2:8], ys[2:8], zs[2:8], ds[2:8], pts[POINT_OF_PLANE], np.array(f.origin[:], np.float64)


def _views(rng, n):
    out = []
    for k in range(n):
        p = rng.normal(size=3) * (2000.0 if k % 3 else 2e5)
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        up = np.cross(np.cross(d, rng.normal(size=3)), d); up /= np.linalg.norm(up)
        if k % 4 == 0:  # axis aligned, camera on a cell corner: planes coincide with cell faces
            p = np.round(p / 300.0) * 300.0
            d, up = np.array([0.0, 0.0, -1.0]), np.array([0.0, 1.0, 0.0])
        far = float(rng.choice([50.0, 1500.0, 4500.0, 50000.0]))
        if k % 5 == 4:
            out.append(lb.frustum_ortho(p, d.astype(F), up.astype(F), float(rng.uniform(20, 4000)), float(rng.uniform(20, 4000)), 0.0, far))
        else:
            out.append(lb.frustum_perspective(p, d.astype(F), up.astype(F), float(rng.uniform(0.2, 2.4)), float(rng.uniform(0.5, 2.5)), float(rng.uniform(0.01, 2.0)), far))
    return out


def _cells_near(rng, origin, n, spread):
    idx = np.round((origin[None, :] + rng.normal(size=(n, 3)) * spread) / 300.0)
    return idx * 300.0  # cell origins (fp64, multiples of 300 like IVec3 * 300.0)


def test_lean_cheap_pass_never_drops_a_page_the_exact_tests_keep():
    rng = np.random.default_rng(11)
    dropped = kept = 0
    for f in _views(rng, 60):
        nx, ny, nz, d, _, org = _planes(f)
        for spread in (600.0, 3000.0, 30000.0):
            cells = _cells_near(rng, org, 4000, spread)
            # exact tests (classify_cell, csrc/cull_common.cuh): float32 op for op
            rel_c = ((cells + np.float64(CS)) - org).astype(F)
            max_c = rel_c + CS
            rel_i = ((cells - np.float64(CS)) - org).astype(F)
            max_i = rel_i + F(2) * CS
            contains = np.ones(len(cells), bool); intersects = np.ones(len(cells), bool); outside_cheap = np.zeros(len(cells), bool)
            for p in range(6):
                nd = -d[p]
                cb = [np.where(n_ < 0, mx, mn) for n_, mx, mn in ((nx[p], max_c[:, 0], rel_c[:, 0]), (ny[p], max_c[:, 1], rel_c[:, 1]), (nz[p], max_c[:, 2], rel_c[:, 2]))]
                dp_c = (nx[p] * cb[0] + ny[p] * cb[1]) + nz[p] * cb[2]
                contains &= ~(dp_c < nd)
                ib = [np.where(n_ > 0, mx, mn) for n_, mx, mn in ((nx[p], max_i[:, 0], rel_i[:, 0]), (ny[p], max_i[:, 1], rel_i[:, 1]), (nz[p], max_i[:, 2], rel_i[:, 2]))]
                tx, ty, tz = nx[p] * ib[0], ny[p] * ib[1], nz[p] * ib[2]
                dp_i = (tx + ty) + tz
                intersects &= ~(dp_i < nd)
                margin = F(1e-4) * (np.abs(nd) + np.abs(tx) + np.abs(ty) + np.abs(tz)) + F(0.05)
                outside_cheap |= (dp_i + margin) < nd
            exact_outside = ~contains & ~intersects
            assert not np.any(outside_cheap & ~exact_outside)  # never drops a page that contains or intersects
            dropped += int(outside_cheap.sum()); kept += int((exact_outside & ~outside_cheap).sum())
    assert dropped > 100_000          # the cheap pass does the bulk of the rejections ...
    assert kept < 0.05 * dropped      # ... and leaves only pages within the margin of a plane to the exact pass


def test_masked_planes_cannot_cull_a_sphere_of_the_cell():
    rng = np.random.default_rng(12)
    masked_any = 0
    for f in _views(rng, 40):
        nx, ny, nz, d, pts, org = _planes(f)
        cells = _cells_near(rng, org, 300, 2500.0)
        for c in cells:
            # plane mask, op for op as in the kernels
            e = F(1.0) + F(1e-6) * max(abs(F(c[0])), abs(F(c[1])), abs(F(c[2])))
            lo = np.array([(F(0.0) if c[k] > 0 else -CS) - e for k in range(3)], F)
            hi = np.array([(F(0.0) if c[k] < 0 else CS) + e for k in range(3)], F)
            offset = (org - c).astype(F)
            need = 0
            rd = np.zeros(6, F)
            for p in range(6):
                q = pts[p] + offset
                dp = -((q[0] * nx[p] + q[1] * ny[p]) + q[2] * nz[p])
                rd[p] = dp
                low = dp + min(nx[p] * lo[0], nx[p] * hi[0]) + min(ny[p] * lo[1], ny[p] * hi[1]) + min(nz[p] * lo[2], nz[p] * hi[2])
                margin = F(1e-5) * (abs(dp) + F(1000.0) * (abs(nx[p]) + abs(ny[p]) + abs(nz[p]))) + F(1e-3)
                if not (low > margin):
                    need |= 1 << p
            if need == 0x3F:
                continue
            masked_any += 1
            # spheres anywhere in the cell as the host bins them: index = trunc(pos / 300) (culling_system.cpp:27), cell-relative fp32 position
            lo_w = np.array([0.0 if c[k] > 0 else -300.0 for k in range(3)])
            hi_w = np.array([0.0 if c[k] < 0 else 300.0 for k in range(3)])
            s = (lo_w + (hi_w - lo_w) * rng.random((400, 3))).astype(F)
            s[:8] = np.array([[a, b, c_] for a in (lo_w[0], hi_w[0]) for b in (lo_w[1], hi_w[1]) for c_ in (lo_w[2], hi_w[2])], F)  # the corners
            r = (rng.random(400) * 300.0).astype(F); r[:8] = 0
            for p in range(6):
                if need & (1 << p):
                    continue
                t = ((s[:, 0] * nx[p] + s[:, 1] * ny[p]) + s[:, 2] * nz[p]) + rd[p]
                t = t - (-r)
                assert not np.any(np.signbit(t)), (c, p)
    assert masked_any > 1000
