"""Pose evaluation + skinning palette + CPU-path skinning on the GPU (replaces AnimationModuleImpl::updateAnimable,
src/animation/animation_module.cpp:439-472, and the palette builds pipeline.cpp:2680-2745 / model.cpp:132-137,103-109).

Data classes mirror the reference's in-memory objects:
  AnimationClip  <- struct Animation after load (src/animation/animation.h:82-118,158-170; animation.cpp:397-493)
  Skeleton       <- Model bones (src/renderer/model.h:154-166,225-244)
  SkinnedMesh    <- Mesh::vertices + Mesh::Skin (model.h:81-84)
`AnimationClip.encode` packs float tracks the way the importer does (SURVEY.md Appendix B) so that synthetic clips have
the reference's bit layout.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import PALETTE_DUAL_QUAT, PALETTE_MATRIX, PALETTE_POSE, check, ptr, vp

ONE_SECOND = 1 << 15  # animation.h:42

TRACK_DTYPE = np.dtype([("bone_index", np.uint16), ("offset_bits", np.uint16), ("bitsizes", np.uint8, 3), ("skipped_channel", np.uint8),
                        ("min", np.float32, 3), ("to_range", np.float32, 3)])
CONST_T_DTYPE = np.dtype([("bone_index", np.uint16), ("pad", np.uint16), ("value", np.float32, 3)])
CONST_R_DTYPE = np.dtype([("bone_index", np.uint16), ("pad", np.uint16), ("value", np.float32, 4)])
assert TRACK_DTYPE.itemsize == 32 and CONST_T_DTYPE.itemsize == 16 and CONST_R_DTYPE.itemsize == 20
SAMPLE_DTYPE = np.dtype([("clip", np.uint32), ("time_ticks", np.uint32), ("weight", np.float32), ("looped", np.uint32)])  # lb200_sample
assert SAMPLE_DTYPE.itemsize == 16
IK_DTYPE = np.dtype([("after", np.uint32), ("leaf_bone", np.uint32), ("bone_count", np.uint32), ("alpha", np.float32), ("target", np.float32, 3),
                     ("reserved", np.uint32)])  # lb200_ik
assert IK_DTYPE.itemsize == 32
ROOT_MOTION_DTYPE = np.dtype([("flags", np.uint32), ("translation_track", np.int32), ("rotation_track", np.int32)])  # lb200_root_motion
assert ROOT_MOTION_DTYPE.itemsize == 12
Y_ROOT_TRANSLATION, XZ_ROOT_TRANSLATION, ROOT_ROTATION = 1, 2, 4  # Animation::Flags, animation.h:73-78


def _pack_frames(per_track_values, bits_per_track):
    """per_track_values: list of uint64[frames] (already combined per track); frame-major bit stream + offsets."""
    n_frames = len(per_track_values[0]) if per_track_values else 0
    offsets = np.concatenate([[0], np.cumsum(bits_per_track)]).astype(np.int64)
    frame_bits = int(offsets[-1])
    total_bits = frame_bits * n_frames
    nbytes = (total_bits + 7) // 8 + 8  # +8 tail padding, animation.cpp:439
    stream = np.zeros(nbytes, np.uint8)
    big = 0
    # python ints as an arbitrary-width bit buffer (clips are small: tens of KB)
    for f in range(n_frames):
        for t, vals in enumerate(per_track_values):
            big |= int(vals[f]) << (f * frame_bits + int(offsets[t]))
    raw = big.to_bytes((total_bits + 7) // 8 if total_bits else 0, "little")
    stream[:len(raw)] = np.frombuffer(raw, np.uint8)
    return stream, offsets[:-1].astype(np.uint16), frame_bits


class AnimationClip:
    def __init__(self, fps, frame_count, translations, const_translations, rotations, const_rotations, translation_stream, rotation_stream,
                 translations_frame_size_bits, rotations_frame_size_bits, flags=0):
        self.fps = float(np.float32(fps))
        self.frame_count = int(frame_count)
        self.translations = np.ascontiguousarray(translations, TRACK_DTYPE)
        self.const_translations = np.ascontiguousarray(const_translations, CONST_T_DTYPE)
        self.rotations = np.ascontiguousarray(rotations, TRACK_DTYPE)
        self.const_rotations = np.ascontiguousarray(const_rotations, CONST_R_DTYPE)
        self.translation_stream = np.ascontiguousarray(translation_stream, np.uint8)
        self.rotation_stream = np.ascontiguousarray(rotation_stream, np.uint8)
        self.translations_frame_size_bits = int(translations_frame_size_bits)
        self.rotations_frame_size_bits = int(rotations_frame_size_bits)
        self.flags = int(flags)  # Animation::m_flags: the root-motion bits of the compiled file's header

    @property
    def length_ticks(self):
        # Animation::getLength(): Time::fromSeconds(m_frame_count / m_fps), animation.h:21-24,128
        return int(np.uint32(np.float32(np.float32(self.frame_count) / np.float32(self.fps)) * np.float32(ONE_SECOND)))

    def rootMotionTracks(self, bone):
        """(translation track, rotation track) of `bone` as Animation::setRootMotionBone resolves them (animation.cpp:223-237): the index of
        the bone's first animated (non-constant) track in `translations` / `rotations`, or -1."""
        t = np.nonzero(self.translations["bone_index"] == bone)[0]
        r = np.nonzero(self.rotations["bone_index"] == bone)[0]
        return (int(t[0]) if len(t) else -1, int(r[0]) if len(r) else -1)

    @staticmethod
    def encode(fps, positions, rotations, pos_bits=(16, 16, 16), rot_bits=(15, 15, 15), const_eps=0.0):
        """positions: f32[frames+1, bones, 3], rotations: unit quats f32[frames+1, bones, 4] (xyzw).  Tracks whose value never
        changes become constant tracks; the rest are quantised like model_importer.cpp:78-116,1591-1593,1681-1732."""
        positions = np.asarray(positions, np.float32)
        rotations = np.asarray(rotations, np.float32)
        n_frames, n_bones = positions.shape[0], positions.shape[1]
        frame_count = n_frames - 1
        t_tracks, ct_tracks, r_tracks, cr_tracks = [], [], [], []
        t_vals, t_bits, r_vals, r_bits = [], [], [], []
        for b in range(n_bones):
            p = positions[:, b, :]
            if np.all(np.abs(p - p[0]) <= const_eps):
                ct_tracks.append((b, 0, p[0]))
            else:
                mn = p.min(axis=0).astype(np.float32)
                mx = p.max(axis=0).astype(np.float32)
                bits = np.array(pos_bits, np.int64)
                rng = np.where(mx > mn, mx - mn, np.float32(1)).astype(np.float64)
                scale = ((1 << bits) - 1).astype(np.float64)
                q = np.floor((p.astype(np.float64) - mn) / rng * scale + 0.5).astype(np.uint64)
                q = np.minimum(q, ((1 << bits) - 1).astype(np.uint64))
                combined = q[:, 0] | (q[:, 1] << np.uint64(bits[0])) | (q[:, 2] << np.uint64(bits[0] + bits[1]))
                to_range = ((mx - mn).astype(np.float64) / scale).astype(np.float32)
                t_tracks.append((b, 0, tuple(int(x) for x in bits), 0, mn, to_range))
                t_vals.append(combined)
                t_bits.append(int(bits.sum()))
            r = rotations[:, b, :]
            if np.all(np.abs(r - r[0]) <= const_eps):
                cr_tracks.append((b, 0, r[0]))
            else:
                skipped = int(np.argmax(np.abs(r).mean(axis=0)))
                keep = [c for c in range(4) if c != skipped]
                v = r[:, keep]
                mn = v.min(axis=0).astype(np.float32)
                mx = v.max(axis=0).astype(np.float32)
                bits = np.array(rot_bits, np.int64)
                rng = np.where(mx > mn, mx - mn, np.float32(1)).astype(np.float64)
                scale = ((1 << bits) - 1).astype(np.float64)
                q = np.floor((v.astype(np.float64) - mn) / rng * scale + 0.5).astype(np.uint64)
                q = np.minimum(q, ((1 << bits) - 1).astype(np.uint64))
                sign = (r[:, skipped] < 0).astype(np.uint64)
                combined = sign | ((q[:, 0] | (q[:, 1] << np.uint64(bits[0])) | (q[:, 2] << np.uint64(bits[0] + bits[1]))) << np.uint64(1))
                to_range = ((mx - mn).astype(np.float64) / scale).astype(np.float32)
                r_tracks.append((b, 0, tuple(int(x) for x in bits), skipped, mn, to_range))
                r_vals.append(combined)
                r_bits.append(int(bits.sum()) + 1)
        t_stream, t_off, t_frame_bits = _pack_frames(t_vals, t_bits) if t_vals else (np.zeros(8, np.uint8), np.zeros(0, np.uint16), 0)
        r_stream, r_off, r_frame_bits = _pack_frames(r_vals, r_bits) if r_vals else (np.zeros(8, np.uint8), np.zeros(0, np.uint16), 0)
        T = np.zeros(len(t_tracks), TRACK_DTYPE)
        for i, (b, _, bits, sk, mn, tr) in enumerate(t_tracks):
            T[i] = (b, t_off[i], bits, sk, mn, tr)
        R = np.zeros(len(r_tracks), TRACK_DTYPE)
        for i, (b, _, bits, sk, mn, tr) in enumerate(r_tracks):
            R[i] = (b, r_off[i], bits, sk, mn, tr)
        CT = np.zeros(len(ct_tracks), CONST_T_DTYPE)
        for i, (b, _, v) in enumerate(ct_tracks):
            CT[i] = (b, 0, v)
        CR = np.zeros(len(cr_tracks), CONST_R_DTYPE)
        for i, (b, _, v) in enumerate(cr_tracks):
            CR[i] = (b, 0, v)
        return AnimationClip(fps, frame_count, T, CT, R, CR, t_stream, r_stream, t_frame_bits, r_frame_bits)

    # ---- compiled .ani image (the file Animation::load reads, src/animation/animation.cpp:397-493) ----
    ANI_MAGIC = 0x5F4C4146  # '_LAF', animation.h:56
    ANI_VERSION = 7         # Version::SKELETON: no skeleton path string in the file (animation.h:64-69)

    def to_ani_bytes(self, bone_hashes, flags=0):
        """Serialise the clip the way the asset compiler does: header, fps, frame count, flags, translation track descriptors
        (BoneNameHash u64, TrackType u8, then value or min / to_range / bitsizes / offset_bits), the translation bit stream, rotation
        descriptors (+ skipped_channel) and the rotation bit stream.  bone_hashes[bone_index] = the bone's name hash."""
        import struct
        out = [struct.pack("<II", self.ANI_MAGIC, self.ANI_VERSION), struct.pack("<fII", self.fps, self.frame_count, flags)]
        out.append(struct.pack("<I", len(self.translations) + len(self.const_translations)))
        tracks = [(int(t["bone_index"]), 0, t) for t in self.const_translations] + [(int(t["bone_index"]), 1, t) for t in self.translations]
        for bone, kind, t in sorted(tracks, key=lambda x: (x[0], x[1])):
            out.append(struct.pack("<QB", int(bone_hashes[bone]), kind))
            if kind == 0:
                out.append(struct.pack("<3f", *t["value"]))
            else:
                out.append(struct.pack("<3f3f3BH", *t["min"], *t["to_range"], *[int(x) for x in t["bitsizes"]], int(t["offset_bits"])))
        n = (self.translations_frame_size_bits * (self.frame_count + 1) + 7) // 8  # animation.cpp:461
        out.append(bytes(self.translation_stream[:n]))
        out.append(struct.pack("<I", len(self.rotations) + len(self.const_rotations)))
        tracks = [(int(t["bone_index"]), 0, t) for t in self.const_rotations] + [(int(t["bone_index"]), 1, t) for t in self.rotations]
        for bone, kind, t in sorted(tracks, key=lambda x: (x[0], x[1])):
            out.append(struct.pack("<QB", int(bone_hashes[bone]), kind))
            if kind == 0:
                out.append(struct.pack("<4f", *t["value"]))
            else:
                out.append(struct.pack("<3f3f3BHB", *t["min"], *t["to_range"], *[int(x) for x in t["bitsizes"]], int(t["offset_bits"]), int(t["skipped_channel"])))
        n = (self.rotations_frame_size_bits * (self.frame_count + 1) + 7) // 8
        out.append(bytes(self.rotation_stream[:n]))
        return b"".join(out)

    @staticmethod
    def from_ani_bytes(data, hash_to_bone):
        """Animation::load (animation.cpp:397-493) + the bone index resolution of Animation::onBeforeReady (:366-395): compiled .ani
        image -> AnimationClip.  hash_to_bone maps a BoneNameHash value to the bone index of the skeleton (Model::getBoneIndex)."""
        import struct
        magic, version = struct.unpack_from("<II", data, 0)
        if magic != AnimationClip.ANI_MAGIC:
            raise ValueError("not a compiled animation ('_LAF' magic missing)")
        if version <= 6 or version > 7:
            raise ValueError(f"animation version {version} not supported (7 = SKELETON without an embedded path)")
        pos = 8
        fps, frame_count, flags = struct.unpack_from("<fII", data, pos); pos += 12
        (n_tr,) = struct.unpack_from("<I", data, pos); pos += 4
        T, CT, t_bits = [], [], 0
        for _ in range(n_tr):
            h, kind = struct.unpack_from("<QB", data, pos); pos += 9
            if kind == 0:
                CT.append((hash_to_bone[h], 0, struct.unpack_from("<3f", data, pos))); pos += 12
            else:
                v = struct.unpack_from("<3f3f3BH", data, pos); pos += 29
                T.append((hash_to_bone[h], v[9], v[6:9], 0, v[0:3], v[3:6]))
                t_bits += sum(v[6:9])
        n = (t_bits * (frame_count + 1) + 7) // 8
        t_stream = np.zeros(n + 8, np.uint8); t_stream[:n] = np.frombuffer(data, np.uint8, n, pos); pos += n
        (n_rot,) = struct.unpack_from("<I", data, pos); pos += 4
        R, CR, r_bits = [], [], 0
        for _ in range(n_rot):
            h, kind = struct.unpack_from("<QB", data, pos); pos += 9
            if kind == 0:
                CR.append((hash_to_bone[h], 0, struct.unpack_from("<4f", data, pos))); pos += 16
            else:
                v = struct.unpack_from("<3f3f3BHB", data, pos); pos += 30
                R.append((hash_to_bone[h], v[9], v[6:9], v[10], v[0:3], v[3:6]))
                r_bits += sum(v[6:9]) + 1  # + sign bit, animation.cpp:484
        n = (r_bits * (frame_count + 1) + 7) // 8
        r_stream = np.zeros(n + 8, np.uint8); r_stream[:n] = np.frombuffer(data, np.uint8, min(n, len(data) - pos), pos)[:n]
        return AnimationClip(fps, frame_count, np.array(T, TRACK_DTYPE), np.array(CT, CONST_T_DTYPE), np.array(R, TRACK_DTYPE), np.array(CR, CONST_R_DTYPE),
                             t_stream, r_stream, t_bits, r_bits, flags)

    def as_struct(self, struct_cls):
        """Fill a ctypes clip struct (lumix_b200 `Clip` or any struct with the same field names); keeps the arrays alive through self."""
        s = struct_cls()
        s.fps = self.fps
        s.frame_count = self.frame_count
        s.translations_frame_size_bits = self.translations_frame_size_bits
        s.rotations_frame_size_bits = self.rotations_frame_size_bits
        s.n_translations = len(self.translations)
        s.n_const_translations = len(self.const_translations)
        s.n_rotations = len(self.rotations)
        s.n_const_rotations = len(self.const_rotations)
        s.translations = self.translations.ctypes.data
        s.const_translations = self.const_translations.ctypes.data
        s.rotations = self.rotations.ctypes.data
        s.const_rotations = self.const_rotations.ctypes.data
        s.translation_stream = self.translation_stream.ctypes.data
        s.rotation_stream = self.rotation_stream.ctypes.data
        if hasattr(s, "translation_stream_bytes"):
            s.translation_stream_bytes = len(self.translation_stream)
            s.rotation_stream_bytes = len(self.rotation_stream)
        return s


def _rotate(q, v):
    """Quat::rotate, float32 numpy (setup-time only; math.cpp:164-175)."""
    qv = q[..., :3]
    uv = np.cross(qv, v).astype(np.float32)
    uuv = np.cross(qv, uv).astype(np.float32)
    return (v + uv * (np.float32(2) * q[..., 3:4]) + uuv * np.float32(2)).astype(np.float32)


def _qmul(a, b):
    x = a[..., 3] * b[..., 0] + b[..., 3] * a[..., 0] + a[..., 1] * b[..., 2] - b[..., 1] * a[..., 2]
    y = a[..., 3] * b[..., 1] + b[..., 3] * a[..., 1] + a[..., 2] * b[..., 0] - b[..., 2] * a[..., 0]
    z = a[..., 3] * b[..., 2] + b[..., 3] * a[..., 2] + a[..., 0] * b[..., 1] - b[..., 0] * a[..., 1]
    w = a[..., 3] * b[..., 3] - a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2]
    return np.stack([x, y, z, w], axis=-1).astype(np.float32)


class Skeleton:
    """parents[i] < i for every non-root bone (model.cpp:381-384).  bind_abs7: absolute bind pose (Bone::transform);
    relative_transform and the inverse bind are derived as Model::parseBones does (model.cpp:389-421)."""

    def __init__(self, parents, bind_abs7):
        self.parents = np.ascontiguousarray(parents, np.int16)
        self.bind_abs7 = np.ascontiguousarray(bind_abs7, np.float32).reshape(-1, 7)
        self.bone_count = len(self.parents)
        nonroot = np.nonzero(self.parents >= 0)[0]
        self.first_nonroot_bone_index = int(nonroot[0]) if len(nonroot) else -1
        pos, rot = self.bind_abs7[:, :3], self.bind_abs7[:, 3:]
        # invert(tr): rot' = conjugated (x,y,z,-w); pos' = rot'.rotate(-pos)   (model.cpp:24-30)
        inv_rot = rot * np.array([1, 1, 1, -1], np.float32)
        inv_pos = _rotate(inv_rot, -pos)
        self.inverse_bind7 = np.ascontiguousarray(np.concatenate([inv_pos, inv_rot], axis=1), np.float32)
        rel = self.bind_abs7.copy()
        for i in range(self.bone_count):
            p = int(self.parents[i])
            if p >= 0:  # relative = inverse_bind(parent) * transform   (model.cpp:411-414, math.cpp:859-861)
                ip, ir = self.inverse_bind7[p, :3], self.inverse_bind7[p, 3:]
                rel[i, :3] = _rotate(ir[None, :], pos[i][None, :])[0] + ip
                rel[i, 3:] = _qmul(ir[None, :], rot[i][None, :])[0]
        self.bind_relative7 = np.ascontiguousarray(rel, np.float32)

    def as_struct(self, struct_cls):
        s = struct_cls()
        s.bone_count = self.bone_count
        s.first_nonroot_bone_index = self.first_nonroot_bone_index
        s.parents = self.parents.ctypes.data
        if hasattr(s, "bind_relative7"):
            s.bind_relative7 = self.bind_relative7.ctypes.data
            s.inverse_bind7 = self.inverse_bind7.ctypes.data
        else:  # structs that name the fields without the 7-float suffix
            s.bind_relative = self.bind_relative7.ctypes.data
            s.inverse_bind = self.inverse_bind7.ctypes.data
        return s


class SkinnedMesh:
    def __init__(self, positions, weights, indices):
        self.positions = np.ascontiguousarray(positions, np.float32).reshape(-1, 3)
        self.weights = np.ascontiguousarray(weights, np.float32).reshape(-1, 4)
        self.indices = np.ascontiguousarray(indices, np.int16).reshape(-1, 4)
        self.n_vertices = len(self.positions)

    def as_struct(self):
        s = _lib.Mesh()
        s.n_vertices = self.n_vertices
        s.positions3 = self.positions.ctypes.data
        s.weights4 = self.weights.ctypes.data
        s.indices4 = self.indices.ctypes.data
        return s


class AnimationSystem:
    """All animables sharing one skeleton (AnimationModule's m_animables, animation_module.h:17-21)."""

    def __init__(self, ctx, skeleton, clips, mesh=None, max_instances=1):
        self.L = _lib.lib()
        self.ctx = ctx
        self.skeleton, self.clips, self.mesh = skeleton, list(clips), mesh
        sk = skeleton.as_struct(_lib.Skeleton)
        arr = (_lib.Clip * len(self.clips))(*[c.as_struct(_lib.Clip) for c in self.clips])
        m = mesh.as_struct() if mesh is not None else None
        h = vp()
        check(self.L.lb200_animation_create(ctx.h, C.byref(sk), arr, C.c_uint32(len(self.clips)), C.byref(m) if m is not None else None,
                                            C.c_uint32(max_instances), C.byref(h)), ctx.h)
        self.h = h
        ctx._adopt(self)
        self.n = 0

    def close(self):
        if self.h:
            self.L.lb200_animation_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def setInstances(self, clip_index, time_ticks):
        c = np.ascontiguousarray(clip_index, np.uint32)
        t = np.ascontiguousarray(time_ticks, np.uint32)
        check(self.L.lb200_animation_set_instances(self.h, ptr(c), ptr(t), C.c_uint32(len(c))), self.ctx.h)
        self.n = len(c)

    def setEntities(self, ids):
        """EntityRef::index of the model instance each instance poses (lb200_animation_set_entities): ids[i] for instance i, negative = none;
        instances at or past len(ids) have none.  SortKeys.buildPalettes finds an entity's pose through this table."""
        e = np.ascontiguousarray(ids, np.int32)
        check(self.L.lb200_animation_set_entities(self.h, ptr(e) if len(e) else None, C.c_uint32(len(e))), self.ctx.h)

    def update(self, time_delta, palette=PALETTE_DUAL_QUAT):
        check(self.L.lb200_animation_update(self.h, C.c_float(time_delta), C.c_uint32(palette)), self.ctx.h)

    @staticmethod
    def updateMany(systems, time_delta, palette=PALETTE_DUAL_QUAT):
        """update(time_delta, palette) of every system in one device pass (lb200_animation_update_many): same results, one launch per
        64 systems.  Entries may be None (refused, as the C call refuses a NULL entry); an empty list launches nothing."""
        L = _lib.lib()
        systems = list(systems)
        arr = (vp * max(len(systems), 1))(*[None if s is None else s.h for s in systems])
        ctx = next((s.ctx.h for s in systems if s is not None), None)
        check(L.lb200_animation_update_many(arr, C.c_uint32(len(systems)), C.c_float(time_delta), C.c_uint32(palette)), ctx)

    def skin(self):
        check(self.L.lb200_animation_skin(self.h), self.ctx.h)

    def setLaunch(self, pose_lanes=0, skin_group=0):
        """Launch shape of later update() / skin() calls: pose lanes per instance (4, 8, 16, 32) and skinning instances per block
        (4, 8, 16); 0 keeps the default (environment switch, else 8).  More than 192 bones run 4 pose lanes as 8."""
        check(self.L.lb200_animation_set_launch(self.h, C.c_int(pose_lanes), C.c_int(skin_group)), self.ctx.h)

    def lastLaunch(self):
        """(pose lanes of the last update, instances per block of the last skin); 0 where none has run."""
        g, s = C.c_int(), C.c_int()
        check(self.L.lb200_animation_get_launch(self.h, C.byref(g), C.byref(s)), self.ctx.h)
        return int(g.value), int(s.value)

    def _get(self, fn, width, first, count, dtype=np.float32):
        count = self.n - first if count is None else count
        out = np.empty((count, self.skeleton.bone_count, width), dtype)
        check(fn(self.h, C.c_uint32(first), C.c_uint32(count), ptr(out)), self.ctx.h)
        return out

    def getDualQuats(self, first=0, count=None):
        return self._get(self.L.lb200_animation_get_dual_quats, 8, first, count)

    def getMatrices(self, first=0, count=None):
        return self._get(self.L.lb200_animation_get_matrices, 16, first, count)

    def getPose(self, first=0, count=None):
        count = self.n - first if count is None else count
        pos = np.empty((count, self.skeleton.bone_count, 3), np.float32)
        rot = np.empty((count, self.skeleton.bone_count, 4), np.float32)
        check(self.L.lb200_animation_get_pose(self.h, C.c_uint32(first), C.c_uint32(count), ptr(pos), ptr(rot)), self.ctx.h)
        return pos, rot

    def setLayers(self, clip_index, time_ticks, weight):
        """Blend layers per instance, arrays [n_instances, n_layers] (None / empty removes them): weighted samples applied in order
        on top of the base clip, Animation::getRelativePose with ctx.weight (animation.cpp:117-204)."""
        if clip_index is None or np.size(clip_index) == 0:
            check(self.L.lb200_animation_set_layers(self.h, C.c_uint32(0), None, None, None), self.ctx.h)
            return
        ci = np.ascontiguousarray(clip_index, np.uint32).reshape(self.n, -1)
        tt = np.ascontiguousarray(time_ticks, np.uint32).reshape(self.n, -1)
        w = np.ascontiguousarray(weight, np.float32).reshape(self.n, -1)
        assert ci.shape == tt.shape == w.shape
        check(self.L.lb200_animation_set_layers(self.h, C.c_uint32(ci.shape[1]), ptr(ci), ptr(tt), ptr(w)), self.ctx.h)

    def setSamples(self, offsets, clip, time_ticks, weight, looped):
        """Sample lists (lb200_animation_set_samples): instance i starts from the bind pose and applies samples offsets[i] .. offsets[i+1]
        in order, each (clip, time in ticks, weight, looped) as the SAMPLE instruction of an animator's blend stack
        (controller.cpp:142-157, 267-293).  len(offsets) - 1 instances; the system is in sample-list mode until setInstances."""
        off = np.ascontiguousarray(offsets, np.uint32)
        assert off.ndim == 1 and len(off) >= 1
        s = np.empty(len(np.atleast_1d(clip)), SAMPLE_DTYPE)
        s["clip"], s["time_ticks"], s["weight"], s["looped"] = clip, time_ticks, weight, looped
        check(self.L.lb200_animation_set_samples(self.h, C.c_uint32(len(off) - 1), ptr(off), ptr(s) if len(s) else None), self.ctx.h)
        self.n = len(off) - 1

    def setStacks(self, offsets, clip, time_ticks, weight, looped, ik_offsets, ik_after, ik_leaf, ik_bones, ik_alpha, ik_target):
        """Blend stacks (lb200_animation_set_stacks): setSamples plus IK ops per instance (CSR ik_offsets), op k running evalIK
        (controller.cpp:166-265) with (leaf bone index, bone count, alpha, model-space target [3]) after the first ik_after[k] samples of
        its instance.  Ops of an instance have non-decreasing ik_after; equal ones run in list order."""
        off = np.ascontiguousarray(offsets, np.uint32)
        assert off.ndim == 1 and len(off) >= 1
        s = np.empty(len(np.atleast_1d(clip)), SAMPLE_DTYPE)
        s["clip"], s["time_ticks"], s["weight"], s["looped"] = clip, time_ticks, weight, looped
        ik_off = np.ascontiguousarray(ik_offsets, np.uint32)
        assert ik_off.shape == off.shape
        ik = np.zeros(len(np.atleast_1d(ik_after)), IK_DTYPE)
        ik["after"], ik["leaf_bone"], ik["bone_count"], ik["alpha"] = ik_after, ik_leaf, ik_bones, ik_alpha
        ik["target"] = np.asarray(ik_target, np.float32).reshape(-1, 3)
        check(self.L.lb200_animation_set_stacks(self.h, C.c_uint32(len(off) - 1), ptr(off), ptr(s) if len(s) else None, ptr(ik_off),
                                                ptr(ik) if len(ik) else None), self.ctx.h)
        self.n = len(off) - 1

    def setRootMotion(self, flags, translation_track, rotation_track):
        """Root motion per clip (lb200_animation_set_root_motion), one entry per clip of the system: Animation::Flags and the clip's
        root-motion tracks (AnimationClip.rootMotionTracks, -1 for none).  The clips are then sampled as the reference samples them after
        Animation::setRootMotionBone; flags 0 or both tracks -1 leave a clip as decoded."""
        rm = np.zeros(len(np.atleast_1d(flags)), ROOT_MOTION_DTYPE)
        rm["flags"], rm["translation_track"], rm["rotation_track"] = flags, translation_track, rotation_track
        check(self.L.lb200_animation_set_root_motion(self.h, C.c_uint32(len(rm)), ptr(rm) if len(rm) else None), self.ctx.h)

    def boneAttachments(self, instance, bone, relative7, parent_transforms, original_scale3):
        """updateBoneAttachment (render_module.cpp:377-405) for a batch: world Transforms of entities attached to posed bones."""
        from .hierarchy import TRANSFORM_DTYPE
        inst = np.ascontiguousarray(instance, np.uint32)
        bn = np.ascontiguousarray(bone, np.uint32)
        rel = np.ascontiguousarray(relative7, np.float32).reshape(-1, 7)
        par = np.ascontiguousarray(parent_transforms, TRANSFORM_DTYPE)
        sc = np.ascontiguousarray(original_scale3, np.float32).reshape(-1, 3)
        assert len(inst) == len(bn) == len(rel) == len(par) == len(sc)
        out = np.empty(len(inst), TRANSFORM_DTYPE)
        check(self.L.lb200_animation_bone_attachments(self.h, C.c_uint32(len(inst)), ptr(inst), ptr(bn), ptr(rel), ptr(par), ptr(sc), ptr(out)), self.ctx.h)
        return out

    def boneAttachmentsDevice(self, n, dev_instance, dev_bone, dev_relative7, dev_parent_transforms, dev_original_scale3, dev_out_transforms):
        """The same with every table in device memory (pointers as ints) and the transforms left there."""
        from ._lib import vp
        check(self.L.lb200_animation_bone_attachments_device(self.h, C.c_uint32(n), vp(dev_instance), vp(dev_bone), vp(dev_relative7), vp(dev_parent_transforms),
                                                             vp(dev_original_scale3), vp(dev_out_transforms)), self.ctx.h)

    def computeRelative(self):
        """Pose::computeRelative (pose.cpp:136-146) of every instance's absolute pose (update with PALETTE_POSE first)."""
        check(self.L.lb200_animation_compute_relative(self.h), self.ctx.h)

    def getRelativePose(self, first=0, count=None):
        count = self.n - first if count is None else count
        pos = np.empty((count, self.skeleton.bone_count, 3), np.float32)
        rot = np.empty((count, self.skeleton.bone_count, 4), np.float32)
        check(self.L.lb200_animation_get_relative_pose(self.h, C.c_uint32(first), C.c_uint32(count), ptr(pos), ptr(rot)), self.ctx.h)
        return pos, rot

    def blendPose(self, other, weight, relative=False):
        """Pose::blend (pose.cpp:30-41) per instance: this system's poses move towards `other`'s by weight."""
        check(self.L.lb200_animation_blend_pose(self.h, other.h, C.c_float(weight), C.c_int(1 if relative else 0)), self.ctx.h)

    def getTimes(self, first=0, count=None):
        count = self.n - first if count is None else count
        out = np.empty(count, np.uint32)
        check(self.L.lb200_animation_get_times(self.h, C.c_uint32(first), C.c_uint32(count), ptr(out)), self.ctx.h)
        return out

    def getSkinned(self, first=0, count=None):
        count = self.n - first if count is None else count
        out = np.empty((count, self.mesh.n_vertices, 3), np.float32)
        check(self.L.lb200_animation_get_skinned(self.h, C.c_uint32(first), C.c_uint32(count), ptr(out)), self.ctx.h)
        return out

    def skinnedChecksum(self):
        v = C.c_uint64()
        check(self.L.lb200_animation_skinned_checksum(self.h, C.byref(v)), self.ctx.h)
        return int(v.value)

    def algorithmic_bytes(self, palette, skin=False):
        return int(self.L.lb200_animation_algorithmic_bytes(self.h, C.c_uint32(palette), C.c_int(1 if skin else 0)))
