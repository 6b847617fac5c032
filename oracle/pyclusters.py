"""TEST INFRASTRUCTURE — ctypes wrappers of the fillClusters restatement (oracle/liboracle_clusters.so, oracle_clusters.c) and of the
reference's own fillClusters code (oracle/_ref/libclusters_shim_b200.so, oracle/build_ref.py).  Both take the same inputs, per
light in light order, and give the same outputs."""
import ctypes as C
import os

import numpy as np

from . import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
RESTATEMENT = os.path.join(HERE, "liboracle_clusters.so")  # made by oracle/Makefile on first use
SHIM = os.path.join(HERE, "_ref", "libclusters_shim_b200.so")

POINT_LIGHT = np.dtype([("color", np.float32, 3), ("intensity", np.float32), ("fov", np.float32), ("attenuation_param", np.float32),
                        ("range", np.float32), ("flags", np.uint32)])
CLUSTER_LIGHT = np.dtype([("pos", np.float32, 3), ("radius", np.float32), ("rot", np.float32, 4), ("color", np.float32, 3),
                          ("attenuation_param", np.float32), ("atlas_idx", np.uint32), ("fov", np.float32), ("padding", np.float32, 2)])
CLUSTER = np.dtype([("offset", np.uint32), ("lights_count", np.uint32), ("env_probes_count", np.uint32), ("refl_probes_count", np.uint32)])
ENV_PROBE = np.dtype([("pos", np.float32, 3), ("pad0", np.float32), ("rot", np.float32, 4), ("inner_range", np.float32, 3), ("pad1", np.float32),
                      ("outer_range", np.float32, 3), ("pad2", np.float32), ("sh_coefs", np.float32, (9, 4))])
REFL_PROBE = np.dtype([("pos", np.float32, 3), ("layer", np.uint32), ("rot", np.float32, 4), ("half_extents", np.float32, 3), ("pad1", np.float32)])
SHADOW = np.dtype([("light_idx", np.uint32), ("priority", np.float32), ("entity", np.int32)])

_libs = {}


def load(which="restatement"):
    """'restatement' (made by oracle/Makefile on first use) or 'shim'; None if the shim has not been built."""
    if which not in _libs:
        path = po.make(os.path.basename(RESTATEMENT)) if which == "restatement" else SHIM
        if not os.path.exists(path):
            return None
        L = C.CDLL(path)
        fn = L.oc_clusters_fill if which == "restatement" else L.ref_clusters_fill
        fn.restype = C.c_uint32
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                       C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                       C.c_void_p, C.c_void_p]
        _libs[which] = fn
    return _libs[which]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cluster_planes(points, w, h):
    """The restatement's xplanes[65], yplanes[65], zplanes[17] (f32[., 4])."""
    L = C.CDLL(po.make(os.path.basename(RESTATEMENT)))
    x, y, z = np.zeros((65, 4), np.float32), np.zeros((65, 4), np.float32), np.zeros((17, 4), np.float32)
    L.oc_cluster_planes(_p(np.ascontiguousarray(points, np.float32)), C.c_int(w), C.c_int(h), _p(x), _p(y), _p(z))
    return x, y, z


def prepare(points, w, h, cam, entities, pos3, rot4, point_lights, atlas, env=None, refl=None, which="restatement", map_cap=1 << 16):
    """The inputs of fill() converted and every output array allocated, map[] with room for map_cap entries.  -> (call, outputs):
    call() makes exactly one call of the library and returns the entries map[] needs (written only up to map_cap); outputs() turns the
    arrays into fill()'s dict after a call whose total fitted."""
    fn = load(which)
    assert fn is not None, f"{which} library not built"
    pts = np.ascontiguousarray(points, np.float32).reshape(24)
    cam = np.ascontiguousarray(cam, np.float64).reshape(3)
    ent = np.ascontiguousarray(entities, np.int32)
    n = len(ent)
    pos3 = np.ascontiguousarray(pos3, np.float64).reshape(n, 3)
    rot4 = np.ascontiguousarray(rot4, np.float32).reshape(n, 4)
    pls = np.ascontiguousarray(point_lights, POINT_LIGHT)
    atl = np.ascontiguousarray(atlas, np.int32)
    env = np.ascontiguousarray(env if env is not None else np.zeros(0, ENV_PROBE), ENV_PROBE)
    refl = np.ascontiguousarray(refl if refl is not None else np.zeros(0, REFL_PROBE), REFL_PROBE)
    size = ((w + 63) // 64, (h + 63) // 64, 16)
    lights = np.zeros(max(n, 1), CLUSTER_LIGHT)
    clusters = np.zeros(size[0] * size[1] * size[2], CLUSTER)
    shadow = np.zeros(64, SHADOW)
    uncast = np.zeros(max(n, 1), np.int32)
    m = np.zeros(max(map_cap, 1), np.int32)
    ns, nu, total = C.c_uint32(), C.c_uint32(), [0]
    args = (_p(pts), w, h, _p(cam), n, _p(ent), _p(pos3), _p(rot4), _p(pls), _p(atl), len(env), _p(env), len(refl), _p(refl),
            _p(lights), _p(clusters), _p(m), map_cap, C.byref(ns), _p(shadow), C.byref(nu), _p(uncast))

    def call():
        total[0] = fn(*args)
        return total[0]

    def outputs():
        assert total[0] <= map_cap
        return dict(lights=lights[:n], clusters=clusters, map=m[:total[0]], shadow=shadow[:ns.value], uncast=uncast[:nu.value], size=size)
    return call, outputs


def fill(points, w, h, cam, entities, pos3, rot4, point_lights, atlas, env=None, refl=None, which="restatement"):
    """fillClusters up to the atlas step for lights given in light order: entities (i32), pos3 (f64[n,3]), rot4 (f32[n,4]),
    point_lights (POINT_LIGHT), atlas (i32, -1 = no entry); env / refl probe arrays (ENV_PROBE / REFL_PROBE) as the host sorted them.
    A map past the first room (65,536 entries) takes a second call with room for all of it.
    -> dict(lights, clusters, map, shadow, uncast, size)."""
    args = (points, w, h, cam, entities, pos3, rot4, point_lights, atlas, env, refl)
    call, outputs = prepare(*args, which=which)
    total = call()
    if total > 1 << 16:
        call, outputs = prepare(*args, which=which, map_cap=total)
        call()
    return outputs()
