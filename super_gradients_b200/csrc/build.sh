#!/usr/bin/env bash
# Builds libsgb200.so (sm_90a only) in-tree.  Usage: build.sh [extra nvcc flags]
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
OUT="$HERE/../libsgb200.so"
OBJ="$HERE/obj"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -I"$ROOT/include" -I"$HERE" --expt-relaxed-constexpr)
mkdir -p "$OBJ"
pids=()
for f in "$HERE"/*.cu; do
  o="$OBJ/$(basename "${f%.cu}").o"
  stale=0
  for h in "$HERE"/*.cuh "$HERE"/*.h "$ROOT/include/sgb200.h" "$HERE/build.sh"; do [[ "$h" -nt "$o" ]] && stale=1; done
  if [[ ! -f "$o" || "$f" -nt "$o" || $stale -eq 1 ]]; then
    "$NVCC" "${FLAGS[@]}" "$@" -c "$f" -o "$o" &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && { wait "$p" || exit 1; }; done
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" "$OBJ"/*.o -lcudart
echo "built $OUT"
