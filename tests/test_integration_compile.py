"""The engine-side bindings under lumixengine_b200/host/ compile against the reference's own sources: the CullingSystem shim
(same vtable, same types, same ownership calls) and the World patch (appended to a temporary copy of world.cpp, as INTEGRATION.md
says a maintainer would).  Only where /root/reference is present (this container)."""
import os
import subprocess
import tempfile

import pytest

from oracle import build_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = build_ref.reference()


def _copy_headers(tmp):
    """The reference files of oracle/build_ref.py's overlay, copied into tmp/src, with its sync.h edit (the Linux port of the reference
    lacks an SRWLock body, src/core/sync.h:22-24, SURVEY F8)."""
    src = os.path.join(tmp, "src")
    build_ref.copy_sources(REF, src)
    build_ref.patch_sync(src)
    return src


GXX = ["/usr/bin/g++", "-std=c++20", "-DSTATIC_PLUGINS", "-DNDEBUG", "-fno-exceptions", "-fno-rtti", "-msse2", "-w", "-c"]


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "engine")), reason="reference tree not present")
def test_world_patch_compiles_inside_world_cpp():
    """host/world_b200_decl.inl goes into `struct World`, host/world_b200.inl is appended to world.cpp: the result must compile with
    the reference's own flags and define World::propagateHierarchyB200 next to the untouched World::transformEntity."""
    with tempfile.TemporaryDirectory() as tmp:
        src = _copy_headers(tmp)
        build_ref.patch_world(src)  # asserts the anchors of INTEGRATION.md section 2
        wc = os.path.join(src, "engine", "world.cpp")
        obj = os.path.join(tmp, "world.o")
        cmd = GXX + ["-I", src, "-I", os.path.join(REF, "external"), "-I", os.path.join(ROOT, "include"), wc, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "Lumix::World::propagateHierarchyB200(lb200_ctx*, bool)" in syms
        assert "Lumix::World::setTransformsDeferredB200(Lumix::EntityRef const*, Lumix::Transform const*, unsigned int)" in syms
        assert "Lumix::World::transformEntity(Lumix::EntityRef, bool)" in syms
        for f in ("lb200_hierarchy_create", "lb200_hierarchy_set_locals", "lb200_hierarchy_propagate", "lb200_hierarchy_get_globals"):
            assert f in syms  # unresolved here, provided by liblumix_b200.so


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "engine")), reason="reference tree not present")
def test_plugin_entry_compiles_against_engine_headers():
    """host/b200_system.cpp: the ISystem + LUMIX_PLUGIN_ENTRY the engine's SystemManager loads (plugin.h:64-96), static-plugin flavour."""
    with tempfile.TemporaryDirectory() as tmp:
        src = _copy_headers(tmp)
        obj = os.path.join(tmp, "b200_system.o")
        cmd = GXX + ["-I", src, "-I", os.path.join(REF, "external"), "-I", os.path.join(ROOT, "include"),
                     os.path.join(ROOT, "lumixengine_b200", "host", "b200_system.cpp"), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "createPlugin_b200" in syms  # -DSTATIC_PLUGINS: the name plugins.inl references
        for f in ("lb200_init", "lb200_shutdown", "lb200_synchronize"):
            assert f in syms


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "renderer")), reason="reference tree not present")
def test_shim_compiles_against_engine_headers():
    with tempfile.TemporaryDirectory() as tmp:
        src = _copy_headers(tmp)  # copied to a temp dir so that sync.h can carry the overlay (never into this repository)
        obj = os.path.join(tmp, "shim.o")
        cmd = GXX + ["-I", src, "-I", os.path.join(REF, "external"), "-I", os.path.join(ROOT, "include"),
                     os.path.join(ROOT, "lumixengine_b200", "host", "culling_system_b200.cpp"), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "Lumix::CullingSystem::create(Lumix::IAllocator&, Lumix::PageAllocator&)" in syms
        assert "lb200_culling_cull" in syms  # unresolved here, provided by liblumix_b200.so


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "animation")), reason="reference tree not present")
def test_animation_binding_compiles_against_render_module():
    """host/animation_b200.inl instantiated with the engine's own RenderModule (render_module.h:402-403 lockPose / unlockPose,
    getModelInstanceModel), animation.h patched with host/animation_b200_decl.inl as INTEGRATION.md section 3 says."""
    host = os.path.join(ROOT, "lumixengine_b200", "host")
    with tempfile.TemporaryDirectory() as tmp:
        src = _copy_headers(tmp)
        patched = os.path.join(tmp, "patched")
        build_ref.patch_animation(src, patched)  # asserts the anchor of INTEGRATION.md section 3
        tu = os.path.join(tmp, "tu.cpp")
        open(tu, "w").write('#include "animation/animation.h"\n#include "animation/animation_module.h"\n#include "core/log.h"\n#include "renderer/model.h"\n'
                            '#include "renderer/pose.h"\n#include "renderer/render_module.h"\n#include <string.h>\n#include "animation_b200.inl"\n'
                            'namespace Lumix { template struct AnimablesB200<RenderModule>; }\n')
        obj = os.path.join(tmp, "tu.o")
        cmd = GXX + ["-I", patched, "-I", src, "-I", os.path.join(REF, "external"), "-I", os.path.join(ROOT, "include"), "-I", host, tu, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "Lumix::AnimablesB200<Lumix::RenderModule>::update(lb200_ctx*, Lumix::RenderModule&, Lumix::Span<Lumix::Animable>, float)" in syms
        for f in ("lb200_animation_create", "lb200_animation_set_instances", "lb200_animation_update", "lb200_animation_get_pose", "lb200_animation_get_times"):
            assert f in syms
