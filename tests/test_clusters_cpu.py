"""The fillClusters restatement (oracle/oracle_clusters.c) against the reference's own fillClusters code (oracle/_ref/libclusters_shim_b200.so,
where it is built) and against tests/golden/clusters_kat.npz, which tests/golden/make_clusters_golden.py makes from that code.  Bytes of
lights[], clusters[], map[], the AtlasSorter list and the uncast-in-atlas list must be equal.

The cases (shared with tests/golden/make_clusters_golden.py): random lights and probes over random perspective and ortho frusta built by
lb200_frustum_from_viewport, lights exactly at dist == +-r of a plane, range 0, lights behind the near plane and beyond the far plane,
viewports of 1x1, 63, 64, 65 and 4096 px, more than 64 casters with equal priorities, and NaN priorities."""
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from oracle import pyclusters as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KAT = os.path.join(ROOT, "tests", "golden", "clusters_kat.npz")
OUTPUTS = ("lights", "clusters", "map", "shadow", "uncast")


def restatement():
    return pc.load("restatement")


def unit_quat(rng):
    q = rng.normal(size=4)
    return (q / np.linalg.norm(q)).astype(np.float32)


def frustum(is_ortho, w, h, cam, rot, fov=1.0472, ortho_size=40.0, near=0.1, far=1000.0):
    """lb200_frustum_from_viewport: (points f32[24], the ShiftedFrustum)."""
    f = lb.frustum_from_viewport(cam, rot, fov, w, h, near, far, is_ortho=is_ortho, ortho_size=ortho_size)
    return np.array([[f.points[i][c] for c in range(3)] for i in range(8)], np.float32).reshape(24), f


def random_probes(rng, n, dtype, extent_field, spread, scale):
    p = np.zeros(n, dtype)
    p["pos"] = (rng.uniform(-spread, spread, (n, 3))).astype(np.float32)
    p["rot"] = np.array([unit_quat(rng) for _ in range(n)]).reshape(n, 4)
    p[extent_field] = rng.uniform(0.1, scale, (n, 3)).astype(np.float32)
    if dtype == pc.ENV_PROBE:
        p["inner_range"] = p["outer_range"] * np.float32(0.5)
        p["sh_coefs"] = rng.normal(size=(n, 9, 4)).astype(np.float32)
    else:
        p["layer"] = np.arange(n, dtype=np.uint32)
    return p


def random_lights(rng, n, cam, spread, r_range=(0.5, 20.0), cast_fraction=0.3, atlas_fraction=0.1):
    """n lights around the camera: entity ids (shuffled, distinct), fp64 positions, rotations, PointLight records, atlas entries."""
    ent = rng.permutation(4 * n + 8)[:n].astype(np.int32)
    pos3 = np.asarray(cam, np.float64) + rng.uniform(-spread, spread, (n, 3))
    rot4 = np.array([unit_quat(rng) for _ in range(n)], np.float32).reshape(n, 4)
    pl = np.zeros(n, pc.POINT_LIGHT)
    pl["color"] = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    pl["intensity"] = rng.uniform(0, 10, n).astype(np.float32)
    pl["fov"] = rng.uniform(0.1, 3.0, n).astype(np.float32)
    pl["attenuation_param"] = rng.uniform(0, 100, n).astype(np.float32)
    pl["range"] = rng.uniform(*r_range, n).astype(np.float32)
    pl["flags"] = (rng.random(n) < cast_fraction).astype(np.uint32) | (2 * (rng.random(n) < 0.5)).astype(np.uint32)
    atlas = np.full(n, -1, np.int32)
    k = rng.random(n) < atlas_fraction
    atlas[k] = rng.integers(0, 37, int(k.sum()))
    return dict(entities=ent, pos3=pos3, rot4=rot4, point_lights=pl, atlas=atlas)


def case(name):
    """Inputs of one named case: dict(points, w, h, cam, entities, pos3, rot4, point_lights, atlas, env, refl)."""
    seed = sum(ord(c) * (i + 1) for i, c in enumerate(name))
    rng = np.random.default_rng(seed)
    cam = tuple(rng.uniform(-1000, 1000, 3))
    rot = unit_quat(rng)
    w, h, ortho, far = 1920, 1080, False, 1000.0
    n, spread, r_range = 300, 200.0, (0.5, 20.0)
    n_env, n_refl = 5, 7
    kw = {}
    if name.startswith("random_ortho"):
        ortho, w, h = True, int(rng.integers(64, 2000)), int(rng.integers(64, 2000))
    elif name.startswith("random_persp"):
        w, h = int(rng.integers(64, 4097)), int(rng.integers(64, 4097))
    elif name.startswith("viewport_"):
        w, h = {"viewport_1x1": (1, 1), "viewport_63": (63, 63), "viewport_64": (64, 64), "viewport_65": (65, 65),
                "viewport_4096": (4096, 4096), "viewport_65x4096": (65, 4096)}[name]
        n = 100
    elif name == "near_far":
        n, far = 200, 300.0
    elif name == "range_zero":
        r_range = (0.0, 0.0)
    points, _ = frustum(ortho, w, h, cam, rot, far=far, **kw)
    L = random_lights(rng, n, cam, spread, r_range)
    env = random_probes(rng, n_env, pc.ENV_PROBE, "outer_range", spread, 30.0)
    refl = random_probes(rng, n_refl, pc.REFL_PROBE, "half_extents", spread, 30.0)
    if name == "near_far":
        # along the view direction: some behind the camera and the near plane, some past the far plane and past the z planes' 10000
        d = -np.cross(points[6:9] - points[0:3], points[3:6] - points[0:3]).astype(np.float64)
        d /= np.linalg.norm(d)
        t = np.concatenate([rng.uniform(-50, 0.1, n // 4), rng.uniform(0.05, 0.2, n // 4), rng.uniform(250, 400, n // 4), rng.uniform(9000, 11000, n - 3 * (n // 4))])
        L["pos3"] = np.asarray(cam) + t[:, None] * d[None, :] + rng.uniform(-3, 3, (n, 3))
    if name == "plane_touch":
        # cam at the origin and float positions, so Vec3(pos - cam) is exact: r = |planeDist| of one plane, dist == r or dist == -r exactly
        cam = (0.0, 0.0, 0.0)
        points, _ = frustum(False, w, h, cam, rot, far=far)
        xp, yp, zp = pc.cluster_planes(points, w, h)
        planes = [xp[:(w + 63) // 64 + 1], yp[:(h + 63) // 64 + 1], zp]
        p = rng.uniform(-spread, spread, (n, 3)).astype(np.float32)
        L["pos3"] = p.astype(np.float64)
        r = np.zeros(n, np.float32)
        for i in range(n):
            axis = planes[i % 3]
            pl = axis[rng.integers(0, len(axis))]
            d = pl[0] * p[i, 0] + pl[1] * p[i, 1] + pl[2] * p[i, 2] + pl[3]
            r[i] = np.abs(np.float32(d))
        L["point_lights"]["range"] = r
    if name == "equal_priorities":
        # 150 casters near the camera at one position with one fov and range: equal priorities above every other caster's, so the list
        # keeps the first 64 pushed
        L["point_lights"]["flags"] &= ~np.uint32(1)
        L["pos3"][:150] = np.asarray(cam) + 2.0
        L["point_lights"]["fov"][:150] = 1.0
        L["point_lights"]["range"][:150] = 50.0
        L["point_lights"]["flags"][:200] |= 1
    if name == "nan_priorities":
        # fov 0 at the camera (0 / 0), fov 0 with an infinite range (0 * inf), interleaved with ordinary casters, more than 64 in all
        L["point_lights"]["flags"] |= 1
        L["pos3"][0:300:7] = cam
        L["point_lights"]["fov"][0:300:7] = 0.0
        L["point_lights"]["fov"][3:300:11] = 0.0
        L["point_lights"]["range"][3:300:11] = np.inf
    return dict(points=points, w=w, h=h, cam=np.asarray(cam, np.float64), env=env, refl=refl, **L)


CASES = ["random_persp_0", "random_persp_1", "random_persp_2", "random_ortho_0", "random_ortho_1", "plane_touch", "range_zero", "near_far",
         "viewport_1x1", "viewport_63", "viewport_64", "viewport_65", "viewport_4096", "viewport_65x4096", "equal_priorities", "nan_priorities"]


def run(c, which="restatement"):
    return pc.fill(c["points"], c["w"], c["h"], c["cam"], c["entities"], c["pos3"], c["rot4"], c["point_lights"], c["atlas"], c["env"], c["refl"], which=which)


def as_bytes(out):
    return {k: np.ascontiguousarray(out[k]).view(np.uint8) for k in OUTPUTS}


def assert_same(got, exp, what):
    g, e = as_bytes(got), as_bytes(exp)
    for k in OUTPUTS:
        assert g[k].shape == e[k].shape and np.array_equal(g[k], e[k]), f"{what}: {k} differs"


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_code(name):
    restatement()
    if pc.load("shim") is None:
        pytest.skip("oracle/_ref/libclusters_shim_b200.so not built (no reference sources)")
    c = case(name)
    assert_same(run(c), run(c, "shim"), name)


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_golden(name):
    restatement()
    if not os.path.exists(KAT):
        pytest.skip("tests/golden/clusters_kat.npz not present")
    kat = np.load(KAT)
    got = as_bytes(run(case(name)))
    for k in OUTPUTS:
        assert np.array_equal(got[k], kat[f"{name}_{k}"]), f"{name}: {k} differs from the fixture"


def test_cases_cover_the_edges():
    """The cases reach what they are named for: touching spheres, equal and NaN priorities, full and partial coverage."""
    restatement()
    out = run(case("equal_priorities"))
    assert len(out["shadow"]) == 64 and (out["shadow"]["priority"][:64] == out["shadow"]["priority"][0]).all()
    assert list(out["shadow"]["light_idx"]) == list(range(64))
    out = run(case("nan_priorities"))
    assert np.isnan(out["shadow"]["priority"]).any() and len(out["shadow"]) == 64
    out = run(case("viewport_4096"))
    assert out["clusters"].shape == (64 * 64 * 16,) and len(out["map"]) > 0
    for name in ("range_zero", "plane_touch", "near_far", "viewport_1x1"):
        out = run(case(name))
        assert len(out["map"]) == int(out["clusters"]["lights_count"].sum() + out["clusters"]["env_probes_count"].sum() + out["clusters"]["refl_probes_count"].sum())
