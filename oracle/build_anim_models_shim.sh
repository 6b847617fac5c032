#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/_ref/libanim_models_shim_b200.so: the animation binding (lumixengine_b200/host/animation_b200.inl) run
# over several real Lumix::Models next to the reference's own updateAnimable (oracle/ref/ref_anim_models_harness.cpp, entry
# ashim_run_models; tests/test_animation_many_gpu.py).  The reference's sources are prepared exactly as build_ref.sh prepares them: this
# script runs build_ref.sh's own overlay steps and compiler flags (its lines from `S="$TMP/src"` to `FL=`) and its patch of animation.h for
# the binding (section (7)), so there is one copy of each.  Like build_ref.sh it copies nothing of the reference into this repository:
# the overlay lives in a mktemp dir that is deleted afterwards.  Skipped without /root/reference or without liblumix_b200.so.
set -euo pipefail
REF=${LUMIX_REFERENCE:-/root/reference}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/_ref"
PRODUCT_DIR="$(cd "$HERE/../lumixengine_b200" && pwd)"
if [ ! -d "$REF/src/core" ]; then
	echo "build_anim_models_shim.sh: $REF not present — keeping prebuilt oracle/_ref as is" >&2
	exit 0
fi
if [ ! -f "$PRODUCT_DIR/liblumix_b200.so" ]; then
	echo "build_anim_models_shim.sh: liblumix_b200.so not built yet — skipped" >&2
	exit 0
fi
mkdir -p "$OUT"
TMP="$(mktemp -d /tmp/lumix_anim_models.XXXXXX)"
trap 'rm -rf "$TMP"' EXIT

OVERLAY="$(sed -n '/^S="\$TMP\/src"$/,/^FL=/p' "$HERE/build_ref.sh")"
PATCH="$(sed -n '/^\tmkdir -p "\$TMP\/patched\/animation"$/,/^PYEOF$/p' "$HERE/build_ref.sh")"
case "$OVERLAY" in *'FL="'*) ;; *) echo "build_anim_models_shim.sh: build_ref.sh has no overlay section to run" >&2; exit 1;; esac
case "$PATCH" in *animation_b200_decl.inl*) ;; *) echo "build_anim_models_shim.sh: build_ref.sh has no animation.h patch to run" >&2; exit 1;; esac
eval "$OVERLAY"
eval "$PATCH"

# the reference objects the animation binding's harness links in build_ref.sh (core, Resource, Pose, Animation) and its stubs
SRCS="core/job_system core/page_allocator core/default_allocator core/arena_allocator core/linux/thread core/linux/sync core/linux/atomic
      core/linux/fibers core/math core/geometry core/string core/hash core/log core/stream core/path engine/resource renderer/pose animation/animation"
OBJS=""
for f in $SRCS; do
	o="$TMP/obj/$(echo "$f" | tr / _).o"
	$CXX $FL -c "$S/$f.cpp" -o "$o" &
	OBJS="$OBJS $o"
done
$CXX $FL -c "$HERE/ref/ref_stubs.cpp" -o "$TMP/obj/ref_stubs.o" &
$CXX -I"$TMP/patched" $FL -I"$HERE/../include" -I"$PRODUCT_DIR/host" -c "$HERE/ref/ref_anim_models_harness.cpp" -o "$TMP/obj/anim_models_harness.o" 2> "$TMP/harness.log" &
wait
# as build_ref.sh does for the engine shim: a harness that does not build is reported and its test skips, the build goes on
if [ -f "$TMP/obj/anim_models_harness.o" ] && $CXX -shared -o "$OUT/libanim_models_shim_b200.so" $OBJS "$TMP/obj/ref_stubs.o" "$TMP/obj/anim_models_harness.o" \
	-L"$PRODUCT_DIR" -llumix_b200 -Wl,-rpath,'$ORIGIN/../../lumixengine_b200' -lpthread -Wl,--no-undefined -Wl,--exclude-libs,ALL 2>> "$TMP/harness.log"; then
	echo "built $OUT/libanim_models_shim_b200.so"
else
	echo "build_anim_models_shim.sh: multi-model animation harness not built (see below)" >&2
	tail -8 "$TMP/harness.log" >&2 || true
fi
