#!/bin/bash
# Build libsetk_b200.so for sm_90a (H100) in-tree.  No GPU needed (nvcc cross-compiles).
# Every csrc/*.cu is one translation unit.  An object is rebuilt when its .cu, any csrc/*.cuh,
# include/setk_b200.h or this script is newer than it.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OUT="$ROOT/setk_b200/libsetk_b200.so"
OBJ="$HERE/obj"
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -I$ROOT/include ${SETK_NVCC_EXTRA}"
DEPS=("$HERE"/*.cuh "$ROOT/include/setk_b200.h" "$HERE/build.sh")
pids=()
objs=()
for src in "$HERE"/*.cu; do
  o="$OBJ/$(basename "$src" .cu).o"
  objs+=("$o")
  stale=0
  [ -f "$o" ] || stale=1
  for d in "$src" "${DEPS[@]}"; do
    [ "$d" -nt "$o" ] && stale=1
  done
  if [ $stale -eq 1 ]; then
    ( $NVCC $FLAGS -Xptxas -v -c "$src" -o "$o.tmp" > "${o%.o}.log" 2>&1 && mv "$o.tmp" "$o" ) &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
if [ $rc -ne 0 ]; then cat "$OBJ"/*.log | grep -v "^ptxas info" | head -100; exit 1; fi
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT" "${objs[@]}"
echo "built $OUT"
