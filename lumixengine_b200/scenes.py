"""Seeded synthetic scenes of the BASELINE.json configs (SURVEY.md §8d C1–C5).  Pure numpy: these are inputs, handed
identically to the GPU path and to whatever checks it.
"""
import numpy as np

from .animation import AnimationClip, SkinnedMesh, Skeleton
from .hierarchy import TRANSFORM_DTYPE

FOV_60 = 1.0472
RATIO_16_9 = 16.0 / 9.0


def cull_scene(n, extent=(2000.0, 200.0, 2000.0), seed=1, big_fraction=0.0, type_probs=(1.0,), radius=(0.5, 5.0)):
    """n spheres uniform in [-ex,ex]x[-ey,ey]x[-ez,ez]; radius U[radius]; `big_fraction` get radius U[300,600] (is_big cells);
    types drawn with `type_probs`.  Returns dict(entities i32, types u8, pos f64[n,3], radius f32)."""
    rng = np.random.default_rng(seed)
    ext = np.asarray(extent, np.float64)
    pos = (rng.random((n, 3), np.float32).astype(np.float64) * 2.0 - 1.0) * ext
    rad = (np.float32(radius[0]) + np.float32(radius[1] - radius[0]) * rng.random(n, np.float32)).astype(np.float32)
    if big_fraction > 0:
        big = rng.random(n) < big_fraction
        rad[big] = (np.float32(300.0) + np.float32(300.0) * rng.random(int(big.sum()), np.float32)).astype(np.float32) + np.float32(0.5)
    probs = np.asarray(type_probs, np.float64)
    types = rng.choice(len(probs), size=n, p=probs / probs.sum()).astype(np.uint8)
    return dict(entities=np.arange(n, dtype=np.int32), types=types, pos=np.ascontiguousarray(pos), radius=rad)


def c1_scene(n=100_000, seed=1):
    """C1: 100 k static spheres, type 0 (MESH); frustum c1_frustum_args()."""
    return cull_scene(n, (2000.0, 200.0, 2000.0), seed)


def c2_scene(n=10_000_000, seed=2):
    """C2: 10 M entities, C1's box scaled x3 (x,z) / x1.5 (y), 0.1 % is_big, 4 renderable types 85/5/5/5 %."""
    return cull_scene(n, (6000.0, 300.0, 6000.0), seed, big_fraction=0.001, type_probs=(0.85, 0.05, 0.05, 0.05))


def c1_frustum_args():
    return dict(position=(0.0, 0.0, 0.0), direction=(0.0, 0.0, -1.0), up=(0.0, 1.0, 0.0), fov=FOV_60, ratio=RATIO_16_9, near=0.1, far=1500.0)


def c2_frustum_args():
    """Same view as C1 with the far plane scaled with the box (x3) so the visible share stays in C1's regime (~15 %)."""
    a = c1_frustum_args()
    a["far"] = 4500.0
    return a


SHADOW_CAM_FAR = 500.0  # pipeline.cpp:270
DEFAULT_CASCADES = (3.0, 10.0, 60.0, 150.0)  # pipeline.cpp:741, without an environment light


def shadow_cascade_args(camera, light_dir, cascades=DEFAULT_CASCADES):
    """Ortho frustum arguments (lb200_frustum_ortho) of the four shadow cascades PipelineImpl::prepareShadowCameras derives for a
    perspective camera given as c1_frustum_args() (pipeline.cpp:734-827): slice i covers the camera's depth range between split
    distances i and i + 1 of (0.1, *cascades); its bounding sphere (Frustum::computeBoundingSphere, geometry.cpp:231-249) sets the size
    bb; the slice's corners projected on xvec / yvec set the ortho size and centre; the camera sits SHADOW_CAM_FAR - 2 bb back along
    the light and sees 0 .. SHADOW_CAM_FAR + 2 bb.  A numpy restatement in float64, for test and timing inputs."""
    unit = lambda v: np.asarray(v, np.float64) / np.linalg.norm(v)  # noqa: E731
    pos = np.asarray(camera["position"], np.float64)
    view_dir, up = unit(camera["direction"]), unit(camera["up"])
    right = unit(np.cross(view_dir, up))
    up = np.cross(right, view_dir)
    light = unit(light_dir)
    xvec = unit(np.cross(light, view_dir))
    yvec = unit(np.cross(light, xvec))
    splits = (0.1,) + tuple(float(c) for c in cascades)
    tan_half = np.tan(camera["fov"] * 0.5)
    out = []
    for s in range(4):
        pts = []
        for dist in (splits[s], splits[s + 1]):
            hh = tan_half * dist
            hw = hh * camera["ratio"]
            for sx in (-1.0, 1.0):
                for sy in (-1.0, 1.0):
                    pts.append(view_dir * dist + right * sx * hw + up * sy * hh)
        pts = np.array(pts)
        bb = float(np.linalg.norm(pts - pts.mean(0), axis=1).max())
        px, py = pts @ xvec, pts @ yvec
        ortho = max(px.max() - px.min(), py.max() - py.min()) * 0.5
        cam = xvec * (px.max() + px.min()) * 0.5 + yvec * (py.max() + py.min()) * 0.5 - light * (SHADOW_CAM_FAR - 2.0 * bb)
        out.append(dict(position=tuple(pos + cam), direction=tuple(light), up=tuple(yvec), width=float(ortho), height=float(ortho), near=0.0,
                        far=SHADOW_CAM_FAR + 2.0 * bb))
    return out


def random_unit_quats(rng, n):
    q = rng.normal(size=(n, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True).astype(np.float32)
    return q.astype(np.float32)


def hierarchy_forest(n_total=1_000_000, depth=8, fanout=7, seed=3, root_extent=(6000.0, 300.0, 6000.0)):
    """C3: forest of complete `fanout`-ary trees of exactly `depth` levels, truncated to n_total nodes.
    Returns parents i32[n], locals TRANSFORM[n], root_globals TRANSFORM[n] (only roots meaningful)."""
    rng = np.random.default_rng(seed)
    per_tree = sum(fanout ** l for l in range(depth))
    n_trees = max(1, n_total // per_tree)
    # node numbering: tree-major, level-major inside a tree
    level_sizes = [fanout ** l for l in range(depth)]
    level_off = np.concatenate([[0], np.cumsum(level_sizes)])
    local_parent = np.full(per_tree, -1, np.int64)
    for l in range(1, depth):
        idx = np.arange(level_sizes[l])
        local_parent[level_off[l] + idx] = level_off[l - 1] + idx // fanout
    parents = (local_parent[None, :] + (np.arange(n_trees, dtype=np.int64) * per_tree)[:, None])
    parents[:, 0] = -1
    parents = parents.reshape(-1)
    n = len(parents)
    if n < n_total:  # pad with extra roots so the node count is exact
        parents = np.concatenate([parents, np.full(n_total - n, -1, np.int64)])
        n = n_total
    locals_ = np.zeros(n, TRANSFORM_DTYPE)
    locals_["pos"] = (rng.random((n, 3)) * 20.0 - 10.0)
    locals_["rot"] = random_unit_quats(rng, n)
    locals_["scale"] = (np.float32(0.8) + np.float32(0.45) * rng.random((n, 3), np.float32)).astype(np.float32)
    globals_ = np.zeros(n, TRANSFORM_DTYPE)
    ext = np.asarray(root_extent, np.float64)
    globals_["pos"] = (rng.random((n, 3)) * 2.0 - 1.0) * ext
    globals_["rot"] = random_unit_quats(rng, n)
    globals_["scale"] = (np.float32(0.8) + np.float32(0.45) * rng.random((n, 3), np.float32)).astype(np.float32)
    return parents.astype(np.int32), locals_, globals_


def skeleton(n_bones=64, seed=4, parents=None):
    """C4 skeleton: root + chains hanging off a 4-ary tree, parent < child.  `parents` gives any other topology instead (parent < child,
    roots first, -1 = root); n_bones is then its length."""
    rng = np.random.default_rng(seed)
    if parents is None:
        parents = np.full(n_bones, -1, np.int16)
        for i in range(1, n_bones):
            parents[i] = (i - 1) // 4 if i < 21 else i - 4  # 4-ary tree for the first 21 bones, then 4 parallel chains
    else:
        parents = np.array(parents, np.int16)
        n_bones = len(parents)
        nonroot = np.nonzero(parents >= 0)[0]
        assert np.all(parents[nonroot] < nonroot), "every parent must come before its child"
        assert len(nonroot) == 0 or np.all(parents[nonroot[0]:] >= 0), "roots must come first"
    rel_pos = (rng.random((n_bones, 3), np.float32) - np.float32(0.5)) * np.float32(0.6)
    rel_rot = random_unit_quats(rng, n_bones)
    from .animation import _qmul, _rotate
    abs7 = np.zeros((n_bones, 7), np.float32)
    for i in range(n_bones):
        p = int(parents[i])
        if p < 0:
            abs7[i, :3], abs7[i, 3:] = rel_pos[i], rel_rot[i]
        else:
            abs7[i, :3] = _rotate(abs7[p, 3:][None], rel_pos[i][None])[0] + abs7[p, :3]
            q = _qmul(abs7[p, 3:][None], rel_rot[i][None])[0]
            abs7[i, 3:] = q / np.float32(np.linalg.norm(q))
    return Skeleton(parents, abs7)


def clip(skel, frames=60, fps=30.0, seed=5, pos_bits=(16, 16, 16), rot_bits=(15, 15, 15), const_fraction=0.25):
    """Synthetic clip: smooth random walk around the bind pose; `const_fraction` of the bones keep constant tracks."""
    rng = np.random.default_rng(seed)
    B = skel.bone_count
    n = frames + 1
    base_p, base_r = skel.bind_relative7[:, :3], skel.bind_relative7[:, 3:]
    t = np.linspace(0, 2 * np.pi, n, dtype=np.float32)[:, None, None]
    amp = (rng.random((1, B, 3), np.float32) * np.float32(0.2))
    phase = rng.random((1, B, 3), np.float32) * np.float32(6.28)
    pos = base_p[None] + amp * np.sin(t + phase)
    dq = rng.normal(size=(1, B, 4)).astype(np.float32) * np.float32(0.35)
    rot = base_r[None] + dq * np.sin(t * np.float32(1.0) + phase[..., :1])
    rot = rot / np.linalg.norm(rot, axis=-1, keepdims=True)
    const = rng.random(B) < const_fraction
    pos[:, const, :] = base_p[None, const, :]
    const_r = rng.random(B) < const_fraction
    rot[:, const_r, :] = base_r[None, const_r, :]
    return AnimationClip.encode(fps, pos.astype(np.float32), rot.astype(np.float32), pos_bits, rot_bits)


def mesh(skel, n_vertices=5000, seed=6):
    """C4 mesh: 4 influences per vertex, weights normalised from u16 (model.cpp:544-547)."""
    rng = np.random.default_rng(seed)
    B = skel.bone_count
    # vertices grouped by the bone they belong to, influences from that bone's neighbourhood (parent, a child, grandparent),
    # as importers emit them: mesh parts are contiguous and skinned to adjacent bones
    home = np.sort(rng.integers(0, B, n_vertices))
    par = np.maximum(skel.parents.astype(np.int64), 0)
    child = np.arange(B)
    for b in range(B - 1, 0, -1):
        child[par[b]] = b  # some child of each bone (itself for leaves)
    idx = np.stack([home, par[home], child[home], par[par[home]]], axis=1)
    w = rng.random((n_vertices, 4)) * np.array([1.0, 0.6, 0.3, 0.1])
    w = w / w.sum(axis=1, keepdims=True)
    w16 = np.round(w * 65535.0).astype(np.uint16)
    weights = (w16.astype(np.float32) / np.float32(65535.0)).astype(np.float32)
    pos = skel.bind_abs7[home, :3] + (rng.random((n_vertices, 3), np.float32) - np.float32(0.5)) * np.float32(0.3)
    return SkinnedMesh(pos.astype(np.float32), weights, idx.astype(np.int16))


def instance_times(n, clips, seed=7):
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(clips), n).astype(np.uint32)
    lengths = np.array([c.length_ticks for c in clips], np.uint32)
    tt = (rng.random(n) * lengths[ci]).astype(np.uint32)
    return ci, tt


def sortkey_setup(n_entities, types, pos, n_models=48, seed=7, skinned_fraction=0.1, moved_fraction=0.02, dirty_fraction=0.002, finite_draw_distance=0.25):
    """Synthetic inputs of PipelineImpl::createSortKeys (pipeline.cpp:3789-4018) for a culling scene: models with 1-4 LODs of 1-3 meshes
    (sort keys allocated one per mesh like Renderer::allocSortKey), four material layers (0 default bucket, 1 depth-sorted bucket, 2 not
    in the view, 3 a second default bucket), per-entity model / lod state / MOVED / dirty flags, decal materials for the DECAL and
    CURVE_DECAL renderables (RenderableTypes 1 and 3), random rotations and scales.  Pure numpy.
    -> dict(models, meshes, model_of, lod, flags, pose_frame, decal_sort_key, decal_layer, transforms, layer_to_bucket, depth_sorted_buckets, max_sort_key)"""
    from .sortkeys import SK_MESH_DTYPE, SK_MODEL_DTYPE
    from .hierarchy import TRANSFORM_DTYPE
    rng = np.random.default_rng(seed)
    models = np.zeros(n_models, SK_MODEL_DTYPE)
    meshes = []
    n_skinned_models = max(1, int(round(n_models * skinned_fraction)))
    for m in range(n_models):
        n_lods = int(rng.integers(1, 5))
        d = np.sort(rng.uniform(80.0, 1500.0, 4)) ** 2  # squared LOD distances (model.h:234)
        dist = np.full(4, np.finfo(np.float32).max, np.float32)
        dist[:n_lods - 1] = d[:n_lods - 1]
        if rng.random() < finite_draw_distance:
            dist[n_lods - 1] = d[3] * 4.0  # beyond it getLODMeshIndices returns an empty LOD: the model is not drawn
        models[m]["lod_distances"] = dist
        models[m]["lod_from"], models[m]["lod_to"] = 0, -1
        models[m]["mesh_base"] = len(meshes)
        skinned = m < n_skinned_models
        at = 0
        for l in range(n_lods):
            k = int(rng.integers(1, 4))
            models[m]["lod_from"][l], models[m]["lod_to"][l] = at, at + k - 1
            for _ in range(k):
                meshes.append((len(meshes), int(rng.integers(1, 5000)), float(l), int(rng.choice([0, 0, 0, 1, 2, 3])), 1 if skinned else 0, 0))
            at += k
        models[m]["mesh_count"] = at
    meshes = np.array(meshes, SK_MESH_DTYPE)
    model_of = rng.integers(0, n_models, n_entities).astype(np.uint32)
    lod = rng.choice(np.array([0.0, 1.0, 2.0, 3.0, 4.0, 0.5, 1.25, 2.9, 3.5], np.float32), n_entities).astype(np.float32)
    flags = np.zeros(n_entities, np.uint8)
    flags[rng.random(n_entities) < moved_fraction] |= 1
    flags[rng.random(n_entities) < dirty_fraction] |= 2
    tr = np.zeros(n_entities, TRANSFORM_DTYPE)
    tr["pos"] = pos
    q = rng.normal(size=(n_entities, 4)).astype(np.float32)
    tr["rot"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    tr["scale"] = rng.uniform(0.5, 2.0, (n_entities, 3)).astype(np.float32)
    return dict(models=models, meshes=meshes, model_of=model_of, lod=lod, flags=flags, pose_frame=np.full(n_entities, 0xffffffff, np.uint32),
                decal_sort_key=rng.integers(0, 2000, n_entities).astype(np.uint32), decal_layer=rng.choice(np.array([0, 1, 2, 3], np.uint8), n_entities).astype(np.uint8),
                transforms=tr, layer_to_bucket=[0, 1, 0xff, 2], depth_sorted_buckets=(1,), max_sort_key=len(meshes) - 1)
