"""TEST INFRASTRUCTURE — builds oracle/_ref/*.so from the reference's OWN sources where they lie (LUMIX_REFERENCE, default
/root/reference; never copied into this repo: the patched overlay lives in a temporary directory that is deleted afterwards).  Does not
run the reference's build system (GENie/MSBuild).  The one recipe for every reference library:

  1. overlay   : the copies; the four edits of SURVEY.md §8(c) — src/core/sync.h (SRWLock body), src/core/linux/sync.cpp (stale
                 Semaphore::signal signature + SRWLock methods), src/core/simd.h (take the SSE branch on GCC), src/core/job_system.cpp
                 (noinline on getWorker(): the reference's TLS guard is MSVC/clang pragmas only; 1 MB fiber stacks as on Windows); the
                 cut-outs of CUTS; the World patch of INTEGRATION.md §2 and a patched second copy of animation.h (§3)
  2. compile   : every reference translation unit of REF_TUS and every harness of HARNESSES once, in parallel; stubs in
                 oracle/ref/ref_stubs.cpp (os::mem*, profiler no-ops, atomics missing on Linux)
  3. link      : the libraries of LIBS

Flags mirror the reference's Linux config (scripts/genie.lua:339-342: -msse2, no FMA, no fast-math) plus -msse3 for _mm_hadd_ps
(simd_math.h:111-119) and -ffp-contract=off to make "no FMA" explicit.  Nothing is built without the reference tree (oracle/_ref is
kept as is); the libraries that link liblumix_b200.so are skipped until it is built; a cut-out whose marker is missing or a harness that
does not compile skips only the libraries that need it.  Everything is rebuilt when an input is newer than oracle/_ref/REFERENCE_COMMIT.

    python3 oracle/build_ref.py [--force]
"""
import glob
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(HERE, "_ref")
HOST = os.path.join(ROOT, "lumixengine_b200", "host")
PRODUCT = os.path.join(ROOT, "lumixengine_b200", "liblumix_b200.so")
CXX = os.environ.get("LUMIX_REF_CXX", "/usr/bin/g++")  # not $CXX: a wrapper there may link libstdc++ statically, which clashes with other C++ libs at exit
CXXFLAGS = ["-std=c++20", "-O2", "-DSTATIC_PLUGINS", "-DNDEBUG", "-fno-exceptions", "-fno-rtti", "-msse2", "-msse3", "-ffp-contract=off", "-fPIC", "-w",
            "-fvisibility=hidden"]
LDFLAGS = ["-lpthread", "-Wl,--no-undefined", "-Wl,--exclude-libs,ALL"]

# the reference's own translation units (src/<tu>.cpp)
REF_TUS = ["renderer/culling_system", "core/job_system", "core/page_allocator", "core/default_allocator", "core/arena_allocator", "core/linux/thread",
           "core/linux/sync", "core/linux/atomic", "core/linux/fibers", "core/math", "core/geometry", "core/string", "core/hash", "core/log",
           "core/stream", "core/path", "engine/resource", "renderer/pose", "animation/animation"]
CORE = REF_TUS[1:]  # job system, allocators, math, geometry, log ...; Resource, Pose, Animation for the animation binding

# Cut out of reference files that need the whole renderer / engine to link, into the overlay: name -> [(overlay file, reference file,
# first line, the line that ends the cut (not copied), a marker the overlay file must then hold)], the lines as `awk '/first/{p=1}
# /end/{p=0} p'` selects them; pieces with the same overlay file are appended.  A missing marker skips the harnesses that include them.
CUTS = {
    # PipelineImpl::computeSkeletonDualQuats (pipeline.cpp, DX12-bound) and the two file-static helpers of model.cpp: evaluateSkin :103-109,
    # computeSkinMatrices :132-137 (oracle/ref/ref_palette_harness.cpp)
    "palette": ("palette harness not built; continuing without ref_skeleton_dual_quats", [
        ("src/renderer/extracted_compute_skeleton_dual_quats.inl", "renderer/pipeline.cpp", r"void computeSkeletonDualQuats\(const ModelInstance\* mi\) \{",
         r"void createCommands\(View& view\)", "computeSkeletonDualQuats"),
        ("src/renderer/extracted_model_statics.inl", "renderer/model.cpp", r"^static Vec3 evaluateSkin\(", r"^Vec3 Model::evalVertexPose\(", None),
        ("src/renderer/extracted_model_statics.inl", "renderer/model.cpp", r"^static void computeSkinMatrices\(", r"^RayCastModelHit Model::castRay\(",
         "computeSkinMatrices")]),
    # the sort-key packers (pipeline.cpp:41-143) and Histogram + radixSort (:4020-4144) (oracle/ref/ref_sortkeys_harness.cpp)
    "sortkeys": ("sort-key harness not built; continuing without ref_radix_sort / ref_make_*", [
        ("src/renderer/extracted_sort_key_packers.inl", "renderer/pipeline.cpp", r"^enum class DrawCommandTypes : u8", r"^struct Indirect \{",
         "makeAutoInstancedSortValue"),
        ("src/renderer/extracted_radix_sort.inl", "renderer/pipeline.cpp", r"^\tstruct Histogram \{", r"^\tvoid viewport\(int x, int y, int w, int h\) override",
         "void radixSort")]),
    # getPose .. evalBlendStack (controller.cpp, evalIK included) and the RuntimeContext constructor (nodes.cpp), next to the patched
    # animation.h (oracle/ref/ref_animators_harness.cpp)
    "animators": ("getPose / evalBlendStack / RuntimeContext moved in the reference; animator harness not built", [
        ("patched/animation/extracted_blend_stack.inl", "animation/controller.cpp", r"^static void getPose\(const anim::RuntimeContext& ctx",
         r"^} // ns Lumix::Anim", r"^void evalBlendStack\("),
        ("patched/animation/extracted_runtime_context.inl", "animation/nodes.cpp", r"^RuntimeContext::RuntimeContext\(Controller& controller, IAllocator& allocator\)",
         r"^void RuntimeContext::setInput\(u32 input_idx, float value\)", "input_runtime")]),
    # fillClusters (pipeline.cpp): AtlasSorter and computeShadowPriority; the ClusterLight / Cluster / ClusterEnvProbe / ClusterReflProbe
    # structs; the plane construction; range(), the for_each_*_pair lambdas and the count / offset / map passes (oracle/ref/ref_clusters_harness.cpp)
    "clusters": ("fillClusters moved in the reference; clusters shim not built", [
        ("src/renderer/extracted_cluster_sorter.inl", "renderer/pipeline.cpp", r"^\tstruct AtlasSorter \{$", r"^\tvoid encodeProceduralGeometry\(View& view\) \{$",
         r"void push\(u32 light_idx"),
        ("src/renderer/extracted_cluster_sorter.inl", "renderer/pipeline.cpp", r"^\tstatic float computeShadowPriority\(",
         r"^\tvoid fillClusters\(DrawStream& stream, const CameraParams& cp\) \{$", "computeShadowPriority"),
        ("src/renderer/extracted_cluster_types.inl", "renderer/pipeline.cpp", r"^\t\tstruct ClusterLight \{$", r"^\t\tArenaAllocator& frame_allocator = ",
         "struct ClusterReflProbe"),
        ("src/renderer/extracted_cluster_planes.inl", "renderer/pipeline.cpp", r"^\t\t\tVec4 xplanes\[65\];$", r"^\t\t\tconst Span<EntityRef> refl_probe_entities",
         r"zplanes\[i\] = makePlane"),
        ("src/renderer/extracted_cluster_binning.inl", "renderer/pipeline.cpp", r"^\t\t\tauto range = \[\]\(const Vec3& p, float r, i32 size, const Vec4\* planes\)\{$",
         r"^\t\t\tbind\(m_cluster_buffers.lights, ", "cluster.offset -= ")]),
}

# the harnesses and the repository's host code: object -> (source, include set, cut-outs it needs).  Include sets: "ref" the overlay,
# "product" + include/lumix_b200.h, "binding" + the patched animation.h in front and lumixengine_b200/host
HARNESSES = {
    "ref_stubs": ("oracle/ref/ref_stubs.cpp", "ref", ()),
    "ref_harness": ("oracle/ref/ref_harness.cpp", "ref", ()),
    "ref_anim_harness": ("oracle/ref/ref_anim_harness.cpp", "ref", ()),
    "ref_palette_harness": ("oracle/ref/ref_palette_harness.cpp", "ref", ("palette",)),
    "ref_sortkeys_harness": ("oracle/ref/ref_sortkeys_harness.cpp", "ref", ("sortkeys",)),
    "ref_clusters_harness": ("oracle/ref/ref_clusters_harness.cpp", "ref", ("clusters",)),
    "ref_engine_shim_harness": ("oracle/ref/ref_engine_shim_harness.cpp", "ref", ()),
    "culling_system_b200": ("lumixengine_b200/host/culling_system_b200.cpp", "product", ()),
    "world_b200": ("{src}/engine/world.cpp", "product", ()),  # the reference's world.cpp with the World patch
    "ref_world_shim_harness": ("oracle/ref/ref_world_shim_harness.cpp", "product", ()),
    "ref_anim_shim_harness": ("oracle/ref/ref_anim_shim_harness.cpp", "binding", ()),
    # includes ref_animators_ik_harness.cpp, ref_animators_harness.cpp, ref_anim_models_harness.cpp and ref_anim_shim_harness.cpp in turn
    "ref_root_motion_harness": ("oracle/ref/ref_root_motion_harness.cpp", "binding", ("animators",)),
}

# output -> (objects, optional objects, links liblumix_b200.so)
LIBS = {
    "libref_lumix.so": (REF_TUS + ["ref_stubs", "ref_harness", "ref_anim_harness"], ["ref_palette_harness", "ref_sortkeys_harness"], False),
    # the executed drop-in boundary: the reference's objects minus its CullingSystemImpl, plus host/culling_system_b200.cpp
    # (CullingSystem::create / CullResult::free over liblumix_b200.so), the patched World and the animation binding
    "libengine_shim_b200.so": (CORE + ["ref_stubs", "culling_system_b200", "ref_engine_shim_harness", "world_b200", "ref_world_shim_harness",
                                       "ref_anim_shim_harness"], [], True),
    "libclusters_shim_b200.so": (["core/math", "core/geometry", "ref_stubs", "ref_clusters_harness"], [], False),
    # the animation binding over several Models, animators' blend stacks, their IK and clips with root motion, next to the reference's own code
    "libanimation_shim_b200.so": (CORE + ["ref_stubs", "ref_root_motion_harness"], [], True),
}


def reference():
    return os.environ.get("LUMIX_REFERENCE", "/root/reference")


def log(msg, tail=None):
    print("build_ref.py: " + msg, file=sys.stderr)
    if tail:
        print("\n".join(tail.splitlines()[-12:]), file=sys.stderr)


def _edit(path, fn):
    with open(path) as f:
        text = f.read()
    with open(path, "w") as f:
        f.write(fn(text))


def copy_sources(ref, src):
    """The reference files the overlay compiles or includes, copied into src (a temporary directory)."""
    for sub in ("engine", "renderer", "animation"):
        os.makedirs(os.path.join(src, sub), exist_ok=True)
        for f in glob.glob(os.path.join(ref, "src", sub, "*.h")):
            shutil.copy(f, os.path.join(src, sub))
    shutil.copytree(os.path.join(ref, "src", "core"), os.path.join(src, "core"))
    shutil.copytree(os.path.join(ref, "src", "renderer", "gpu"), os.path.join(src, "renderer", "gpu"))
    for f in ("renderer/culling_system.cpp", "renderer/pose.cpp", "animation/animation.cpp", "engine/resource.cpp", "engine/world.cpp"):
        shutil.copy(os.path.join(ref, "src", f), os.path.join(src, f))


def patch_sync(src):
    """(1) sync.h: SRWLock has no Linux body."""
    _edit(os.path.join(src, "core", "sync.h"), lambda t: t.replace('#error "Not implemented"', "pthread_rwlock_t lock;"))


def patch_core(src):
    """(2)-(4) of the overlay."""
    # (2) linux/sync.cpp: stale signature + missing SRWLock methods
    _edit(os.path.join(src, "core", "linux", "sync.cpp"), lambda t: re.sub(r"^void Semaphore::signal\(\)", "void Semaphore::signal(u32)", t, flags=re.M) + (
        "namespace Lumix {\n"
        "SRWLock::SRWLock() { pthread_rwlock_init(&lock, nullptr); }\n"
        "SRWLock::~SRWLock() { pthread_rwlock_destroy(&lock); }\n"
        "void SRWLock::enterExclusive() { pthread_rwlock_wrlock(&lock); }\n"
        "void SRWLock::exitExclusive() { pthread_rwlock_unlock(&lock); }\n"
        "void SRWLock::enterShared() { pthread_rwlock_rdlock(&lock); }\n"
        "void SRWLock::exitShared() { pthread_rwlock_unlock(&lock); }\n"
        "}\n"))

    # (3) simd.h: use the SSE (MSVC) branch on GCC; GCC's __m128 already has + - * built in, so the overloads of that branch must go
    #     (unary minus then differs from the reference's 0-a only in the sign of zero)
    def sse_on_gcc(text):
        L = text.split("\n")
        out, i, seen_else, in_sse = [], 0, False, False
        while i < len(L):
            line = L[i]
            in_sse = in_sse or "using float4 = __m128;" in line
            seen_else = seen_else or (in_sse and line.strip().startswith("#else"))
            if line.startswith("#if defined _WIN32 && !defined __clang__"):
                line = "#if 1"
            elif "#include <intrin.h>" in line:
                line = "\t#include <immintrin.h>\n\t#include <math.h>\n\t#include <string.h>"
            elif not seen_else and "LUMIX_FORCE_INLINE float4 operator" in line:
                i += 3
                if i < len(L) and L[i].strip() == "":
                    i += 1
                continue
            out.append(line)
            i += 1
        return "\n".join(out)
    _edit(os.path.join(src, "core", "simd.h"), sse_on_gcc)

    # (4) job_system.cpp: keep getWorker() out of line so &g_worker is recomputed after a fiber switch, and give fibers 1 MB of stack:
    #     Windows fibers reserve 1 MB whatever CreateFiber is asked to commit, the Linux port mallocs exactly the 64 KB it is asked for,
    #     which PipelineImpl::radixSort's two 48 KB histograms overflow (ref_sortkeys_harness.cpp runs it in a job)
    _edit(os.path.join(src, "core", "job_system.cpp"), lambda t: re.sub(
        r"^WorkerTask\* getWorker\(\)", "__attribute__((noinline)) WorkerTask* getWorker()", t, flags=re.M).replace(
        "Fiber::create(64 * 1024, manage, new_fiber)", "Fiber::create(1024 * 1024, manage, new_fiber)"))


def patch_world(src):
    """The World patch as INTEGRATION.md section 2 describes it, on the overlay's world.h / world.cpp: the declarations of
    host/world_b200_decl.inl into `struct World`, host/world_b200.inl appended to world.cpp, one line in ~World."""
    anchor = "private:\n\tvoid transformEntity(EntityRef entity, bool update_local);"
    with open(os.path.join(HOST, "world_b200_decl.inl")) as f:
        decl = f.read()

    def header(t):
        assert anchor in t, "world.h changed: INTEGRATION.md section 2 needs another anchor"
        assert "namespace Lumix {" in t
        return t.replace(anchor, decl + anchor).replace("namespace Lumix {", "struct lb200_ctx; // include/lumix_b200.h\nnamespace Lumix {", 1)
    _edit(os.path.join(src, "engine", "world.h"), header)
    dtor = "World::~World() {\n"
    with open(os.path.join(HOST, "world_b200.inl")) as f:
        body = f.read()

    def source(t):
        assert dtor in t, "world.cpp changed: INTEGRATION.md section 2 needs another anchor"
        return t.replace(dtor, dtor + "\tdestroyHierarchyB200();\n", 1) + "\n" + body
    _edit(os.path.join(src, "engine", "world.cpp"), source)


def patch_animation(src, patched):
    """The animation binding (INTEGRATION.md section 3): the accessors of host/animation_b200_decl.inl go into `struct Animation` of a
    second copy of animation.h, patched/animation/animation.h, that only the binding's harnesses see (inline getters: the layout of
    Animation does not change, the reference's own animation.o is compiled from the unpatched header); controller.h beside it, so that
    its #include "animation.h" finds the patched copy."""
    anchor = "\tconst Array<TranslationTrack>& getTranslations() const { return m_translations; }"
    dst = os.path.join(patched, "animation")
    os.makedirs(dst, exist_ok=True)
    with open(os.path.join(src, "animation", "animation.h")) as f:
        t = f.read()
    assert anchor in t, "animation.h changed: INTEGRATION.md section 3 needs another anchor"
    with open(os.path.join(HOST, "animation_b200_decl.inl")) as f:
        decl = f.read()
    with open(os.path.join(dst, "animation.h"), "w") as f:
        f.write(t.replace(anchor, decl + anchor))
    shutil.copy(os.path.join(src, "animation", "controller.h"), dst)


def cut_out(ref, tmp):
    """Write every cut-out of CUTS into the overlay; -> the names of those whose markers are all there."""
    for _, pieces in CUTS.values():
        for dst, src, first, end, _ in pieces:
            lines, on = [], False
            with open(os.path.join(ref, "src", src)) as f:
                for line in f:
                    on = (on or re.search(first, line) is not None) and re.search(end, line) is None
                    if on:
                        lines.append(line)
            with open(os.path.join(tmp, dst), "a") as f:
                f.write("".join(lines))
    def holds(dst, marker):
        with open(os.path.join(tmp, dst)) as f:
            return marker is None or re.search(marker, f.read(), re.M) is not None
    ok = {name for name, (_, pieces) in CUTS.items() if all(holds(dst, marker) for dst, _, _, _, marker in pieces)}
    for name in CUTS.keys() - ok:
        log(CUTS[name][0])
    return ok


def inputs():
    return ([__file__, PRODUCT, os.path.join(ROOT, "include", "lumix_b200.h")] + glob.glob(os.path.join(HERE, "ref", "*"))
            + glob.glob(os.path.join(HOST, "*")))


def up_to_date():
    stamp = os.path.join(OUT, "REFERENCE_COMMIT")
    if not os.path.exists(stamp) or not os.path.exists(os.path.join(OUT, "libref_lumix.so")):
        return False
    return all(os.path.getmtime(f) <= os.path.getmtime(stamp) for f in inputs() if os.path.exists(f))


def build(force=False):
    ref = reference()
    if not os.path.isdir(os.path.join(ref, "src", "core")):
        log(f"{ref} not present — keeping prebuilt oracle/_ref as is")
        return
    if not force and up_to_date():
        return
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory(prefix="lumix_ref_overlay.") as tmp:
        src, patched, obj = (os.path.join(tmp, d) for d in ("src", "patched", "obj"))
        os.makedirs(obj)
        copy_sources(ref, src)
        patch_sync(src)
        patch_core(src)
        patch_world(src)
        patch_animation(src, patched)
        cuts = cut_out(ref, tmp)

        fl = CXXFLAGS + ["-I" + src, "-I" + os.path.join(ref, "external")]
        include = ["-I" + os.path.join(ROOT, "include")]
        flags = {"ref": fl, "product": fl + include, "binding": ["-I" + patched] + fl + include + ["-I" + HOST]}
        jobs = {tu: (os.path.join(src, tu + ".cpp"), fl) for tu in REF_TUS}
        jobs.update({name: (os.path.join(ROOT, s.format(src=src)), flags[inc]) for name, (s, inc, need) in HARNESSES.items() if set(need) <= cuts})

        def path(name):
            return os.path.join(obj, name.replace("/", "_") + ".o")

        def compile_one(name):
            source, cxxflags = jobs[name]
            return name, subprocess.run([CXX] + cxxflags + ["-c", source, "-o", path(name)], capture_output=True, text=True)
        with ThreadPoolExecutor(os.cpu_count()) as pool:
            failed = {name: r.stderr for name, r in pool.map(compile_one, jobs) if r.returncode != 0}
        for name, err in failed.items():
            log(f"{name} did not compile", err)
        if any(tu in failed for tu in REF_TUS):
            raise RuntimeError("a reference translation unit did not compile (see above)")

        built = set()
        for lib, (objs, optional, product) in LIBS.items():
            missing = [o for o in objs + optional if o not in jobs or o in failed]
            if product and not os.path.exists(PRODUCT):
                log(f"liblumix_b200.so not built yet — {lib} skipped")
                continue
            if set(missing) - set(optional):
                log(f"{lib} not built: {', '.join(missing)} missing (see above)")
                continue
            if missing:
                log(f"{lib}: {', '.join(missing)} missing (see above), linked without")
            cmd = [CXX, "-shared", "-o", os.path.join(OUT, lib)] + [path(o) for o in objs + optional if o not in missing]
            if product:
                cmd += ["-L" + os.path.dirname(PRODUCT), "-llumix_b200", "-Wl,-rpath,$ORIGIN/../../lumixengine_b200"]
            r = subprocess.run(cmd + LDFLAGS, capture_output=True, text=True)
            if r.returncode != 0:
                log(f"{lib} did not link", r.stderr)
                continue
            built.add(lib)
            print(f"built {os.path.join(OUT, lib)}")
    if "libref_lumix.so" not in built:
        raise RuntimeError("libref_lumix.so not built (see above)")
    commit = subprocess.run(["git", "rev-parse", "HEAD"], cwd=ref, capture_output=True, text=True)
    with open(os.path.join(OUT, "REFERENCE_COMMIT"), "w") as f:
        f.write((commit.stdout if commit.returncode == 0 else "unknown\n"))


if __name__ == "__main__":
    build(force="--force" in sys.argv[1:])
