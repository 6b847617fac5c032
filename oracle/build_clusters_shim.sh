#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/_ref/libclusters_shim_b200.so: the reference's own fillClusters code (pipeline.cpp) run by
# oracle/ref/ref_clusters_harness.cpp (entry ref_clusters_fill; tests/test_clusters_cpu.py, tests/golden/make_clusters_golden.py).  The
# reference's sources are prepared exactly as build_ref.sh prepares them (its overlay steps and compiler flags are run from build_ref.sh
# itself).  Cut out of pipeline.cpp between marker lines, into the overlay (pipeline.cpp needs the whole renderer to link): AtlasSorter and
# computeShadowPriority; the ClusterLight / Cluster / ClusterEnvProbe / ClusterReflProbe structs; the plane construction; range(), the
# for_each_*_pair lambdas and the count / offset / map passes.  Nothing of the reference is copied into this repository.  Skipped
# without /root/reference.
set -euo pipefail
REF=${LUMIX_REFERENCE:-/root/reference}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/_ref"
if [ ! -d "$REF/src/core" ]; then
	echo "build_clusters_shim.sh: $REF not present — keeping prebuilt oracle/_ref as is" >&2
	exit 0
fi
mkdir -p "$OUT"
TMP="$(mktemp -d /tmp/lumix_clusters.XXXXXX)"
trap 'rm -rf "$TMP"' EXIT

OVERLAY="$(sed -n '/^S="\$TMP\/src"$/,/^FL=/p' "$HERE/build_ref.sh")"
case "$OVERLAY" in *'FL="'*) ;; *) echo "build_clusters_shim.sh: build_ref.sh has no overlay section to run" >&2; exit 1;; esac
eval "$OVERLAY"

P="$REF/src/renderer/pipeline.cpp"
R="$S/renderer"
awk '/^\tstruct AtlasSorter \{$/{p=1} /^\tvoid encodeProceduralGeometry\(View& view\) \{$/{p=0} p' "$P" > "$R/extracted_cluster_sorter.inl"
awk '/^\tstatic float computeShadowPriority\(/{p=1} /^\tvoid fillClusters\(DrawStream& stream, const CameraParams& cp\) \{$/{p=0} p' "$P" >> "$R/extracted_cluster_sorter.inl"
awk '/^\t\tstruct ClusterLight \{$/{p=1} /^\t\tArenaAllocator& frame_allocator = /{p=0} p' "$P" > "$R/extracted_cluster_types.inl"
awk '/^\t\t\tVec4 xplanes\[65\];$/{p=1} /^\t\t\tconst Span<EntityRef> refl_probe_entities/{p=0} p' "$P" > "$R/extracted_cluster_planes.inl"
awk '/^\t\t\tauto range = \[\]\(const Vec3& p, float r, i32 size, const Vec4\* planes\)\{$/{p=1} /^\t\t\tbind\(m_cluster_buffers.lights, /{p=0} p' "$P" > "$R/extracted_cluster_binning.inl"
if ! grep -q "void push(u32 light_idx" "$R/extracted_cluster_sorter.inl" || ! grep -q "computeShadowPriority" "$R/extracted_cluster_sorter.inl" \
	|| ! grep -q "struct ClusterReflProbe" "$R/extracted_cluster_types.inl" || ! grep -q "zplanes\[i\] = makePlane" "$R/extracted_cluster_planes.inl" \
	|| ! grep -q "cluster.offset -= " "$R/extracted_cluster_binning.inl"; then
	echo "build_clusters_shim.sh: fillClusters moved in the reference; clusters shim not built" >&2
	exit 0
fi

SRCS="core/math core/geometry"
OBJS=""
for f in $SRCS; do
	o="$TMP/obj/$(echo "$f" | tr / _).o"
	$CXX $FL -c "$S/$f.cpp" -o "$o" &
	OBJS="$OBJS $o"
done
$CXX $FL -c "$HERE/ref/ref_stubs.cpp" -o "$TMP/obj/ref_stubs.o" &
$CXX $FL -c "$HERE/ref/ref_clusters_harness.cpp" -o "$TMP/obj/clusters_harness.o" 2> "$TMP/harness.log" &
wait
if [ -f "$TMP/obj/clusters_harness.o" ] && $CXX -shared -o "$OUT/libclusters_shim_b200.so" $OBJS "$TMP/obj/ref_stubs.o" "$TMP/obj/clusters_harness.o" \
	-lpthread -Wl,--no-undefined -Wl,--exclude-libs,ALL -lm 2>> "$TMP/harness.log"; then
	echo "built $OUT/libclusters_shim_b200.so"
else
	echo "build_clusters_shim.sh: clusters shim not built (see below)" >&2
	tail -20 "$TMP/harness.log" >&2 || true
fi
