#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/liboracle_ik.so: the IK restatement of animators' blend stacks (oracle/oracle_ik.c) over the pose
# restatement of oracle/liboracle_lumix.so (built first by oracle/Makefile), with the same compiler flags (SSE2 only, no FMA, no fast-math).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/liboracle_ik.so"
if [ -f "$OUT" ] && [ "$OUT" -nt "$HERE/oracle_ik.c" ] && [ "$OUT" -nt "$HERE/oracle.h" ] && [ "$OUT" -nt "$HERE/oracle_math.h" ] && [ "$OUT" -nt "$HERE/liboracle_lumix.so" ]; then
	exit 0
fi
/usr/bin/gcc -std=c11 -O2 -msse2 -ffp-contract=off -fno-fast-math -fPIC -Wall -Wextra -Wno-unused-function -shared -o "$OUT" "$HERE/oracle_ik.c" \
	-L"$HERE" -loracle_lumix -Wl,-rpath,'$ORIGIN' -lm
