#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/_ref/libroot_motion_shim_b200.so: the IK animator harness over clips whose root motion the
# reference's own Animation::setRootMotionBone set (oracle/ref/ref_root_motion_harness.cpp, which includes
# oracle/ref/ref_animators_ik_harness.cpp; entries ref_rm_tables, ref_rm_pose_stack, ref_rm_math, ashim_run_animables_rm,
# ashim_run_animators_rm; tests/test_animation_root_motion_cpu.py, tests/test_animation_root_motion_binding_gpu.py,
# tests/golden/make_root_motion_golden.py).  The reference is prepared exactly as oracle/build_animators_ik_shim.sh prepares it: build_ref.sh's
# overlay steps, compiler flags and animation.h patch, and getPose .. evalBlendStack (controller.cpp) and the RuntimeContext constructor
# (nodes.cpp) cut out between their signature lines at build time; nothing of the reference is copied into this repository.
# Skipped without /root/reference or without liblumix_b200.so.
set -euo pipefail
REF=${LUMIX_REFERENCE:-/root/reference}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/_ref"
PRODUCT_DIR="$(cd "$HERE/../lumixengine_b200" && pwd)"
if [ ! -d "$REF/src/core" ]; then
	echo "build_root_motion_shim.sh: $REF not present — keeping prebuilt oracle/_ref as is" >&2
	exit 0
fi
if [ ! -f "$PRODUCT_DIR/liblumix_b200.so" ]; then
	echo "build_root_motion_shim.sh: liblumix_b200.so not built yet — skipped" >&2
	exit 0
fi
mkdir -p "$OUT"
TMP="$(mktemp -d /tmp/lumix_root_motion.XXXXXX)"
trap 'rm -rf "$TMP"' EXIT

OVERLAY="$(sed -n '/^S="\$TMP\/src"$/,/^FL=/p' "$HERE/build_ref.sh")"
PATCH="$(sed -n '/^\tmkdir -p "\$TMP\/patched\/animation"$/,/^PYEOF$/p' "$HERE/build_ref.sh")"
case "$OVERLAY" in *'FL="'*) ;; *) echo "build_root_motion_shim.sh: build_ref.sh has no overlay section to run" >&2; exit 1;; esac
case "$PATCH" in *animation_b200_decl.inl*) ;; *) echo "build_root_motion_shim.sh: build_ref.sh has no animation.h patch to run" >&2; exit 1;; esac
eval "$OVERLAY"
eval "$PATCH"

# controller.h next to the patched animation.h, so that its #include "animation.h" finds the patched copy; the cut-outs beside them
P="$TMP/patched/animation"
cp "$S/animation/controller.h" "$P/"
awk '/^static void getPose\(const anim::RuntimeContext& ctx/{p=1} /^} \/\/ ns Lumix::Anim/{p=0} p' "$REF/src/animation/controller.cpp" > "$P/extracted_blend_stack.inl"
awk '/^RuntimeContext::RuntimeContext\(Controller& controller, IAllocator& allocator\)/{p=1} /^void RuntimeContext::setInput\(u32 input_idx, float value\)/{p=0} p' \
	"$REF/src/animation/nodes.cpp" > "$P/extracted_runtime_context.inl"
if ! grep -q "^void evalBlendStack(" "$P/extracted_blend_stack.inl" || ! grep -q "input_runtime" "$P/extracted_runtime_context.inl"; then
	echo "build_root_motion_shim.sh: getPose / evalBlendStack / RuntimeContext moved in the reference; animator harness not built" >&2
	exit 0
fi

SRCS="core/job_system core/page_allocator core/default_allocator core/arena_allocator core/linux/thread core/linux/sync core/linux/atomic
      core/linux/fibers core/math core/geometry core/string core/hash core/log core/stream core/path engine/resource renderer/pose animation/animation"
OBJS=""
for f in $SRCS; do
	o="$TMP/obj/$(echo "$f" | tr / _).o"
	$CXX $FL -c "$S/$f.cpp" -o "$o" &
	OBJS="$OBJS $o"
done
$CXX $FL -c "$HERE/ref/ref_stubs.cpp" -o "$TMP/obj/ref_stubs.o" &
$CXX -I"$TMP/patched" $FL -I"$HERE/../include" -I"$PRODUCT_DIR/host" -c "$HERE/ref/ref_root_motion_harness.cpp" -o "$TMP/obj/animators_harness.o" 2> "$TMP/harness.log" &
wait
if [ -f "$TMP/obj/animators_harness.o" ] && $CXX -shared -o "$OUT/libroot_motion_shim_b200.so" $OBJS "$TMP/obj/ref_stubs.o" "$TMP/obj/animators_harness.o" \
	-L"$PRODUCT_DIR" -llumix_b200 -Wl,-rpath,'$ORIGIN/../../lumixengine_b200' -lpthread -Wl,--no-undefined -Wl,--exclude-libs,ALL 2>> "$TMP/harness.log"; then
	echo "built $OUT/libroot_motion_shim_b200.so"
else
	echo "build_root_motion_shim.sh: animator harness not built (see below)" >&2
	tail -20 "$TMP/harness.log" >&2 || true
fi
