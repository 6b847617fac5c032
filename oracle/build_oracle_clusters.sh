#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/liboracle_clusters.so: the fillClusters restatement (oracle/oracle_clusters.c), with the compiler
# flags of oracle/Makefile (SSE2 only, no FMA, no fast-math).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/liboracle_clusters.so"
if [ -f "$OUT" ] && [ "$OUT" -nt "$HERE/oracle_clusters.c" ]; then
	exit 0
fi
/usr/bin/gcc -std=c11 -O2 -msse2 -ffp-contract=off -fno-fast-math -fPIC -Wall -Wextra -Wno-unused-function -shared -o "$OUT" "$HERE/oracle_clusters.c" -lm
