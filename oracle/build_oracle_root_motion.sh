#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/liboracle_root_motion.so: the root-motion restatement (oracle/oracle_root_motion.c) over the pose
# restatement of oracle/liboracle_lumix.so (oracle/Makefile) and the IK restatement of oracle/liboracle_ik.so (oracle/build_oracle_ik.sh),
# both built first, with the same compiler flags (SSE2 only, no FMA, no fast-math).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/liboracle_root_motion.so"
if [ -f "$OUT" ] && [ "$OUT" -nt "$HERE/oracle_root_motion.c" ] && [ "$OUT" -nt "$HERE/oracle.h" ] && [ "$OUT" -nt "$HERE/oracle_math.h" ] \
	&& [ "$OUT" -nt "$HERE/liboracle_lumix.so" ] && [ "$OUT" -nt "$HERE/liboracle_ik.so" ]; then
	exit 0
fi
/usr/bin/gcc -std=c11 -O2 -msse2 -ffp-contract=off -fno-fast-math -fPIC -Wall -Wextra -Wno-unused-function -shared -o "$OUT" "$HERE/oracle_root_motion.c" \
	-L"$HERE" -loracle_ik -loracle_lumix -Wl,-rpath,'$ORIGIN' -lm
