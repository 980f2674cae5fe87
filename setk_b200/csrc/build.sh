#!/bin/bash
# Build libsetk_b200.so for sm_90a (H100) in-tree.  No GPU needed (nvcc cross-compiles).
# Objects are rebuilt only when their .cu or any header is newer.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OUT="$ROOT/setk_b200/libsetk_b200.so"
OBJ="$HERE/obj"
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -I$ROOT/include ${SETK_NVCC_EXTRA}"
# headers each translation unit depends on
declare -A DEPS
DEPS[api]="common.cuh compat.cuh"
DEPS[generic]="common.cuh compat.cuh"
DEPS[weights]="common.cuh compat.cuh hermitian_solve.cuh weights_args.cuh"
DEPS[weights_coop]="common.cuh compat.cuh hermitian_solve.cuh jacobi_coop.cuh lu_coop.cuh weights_args.cuh"
DEPS[weights_post]="common.cuh compat.cuh hermitian_solve.cuh"
DEPS[stft_cov_fused]="common.cuh compat.cuh stft_tile.cuh fft16.cuh async_copy.cuh stft_cov_args.cuh"
DEPS[stft_cov_ws]="common.cuh compat.cuh stft_tile.cuh fft16.cuh async_copy.cuh stft_cov_args.cuh"
DEPS[apply_istft_fused]="common.cuh compat.cuh stft_tile.cuh fft16.cuh async_copy.cuh apply_istft_args.cuh"
DEPS[stft_spill]="common.cuh compat.cuh stft_tile.cuh fft16.cuh async_copy.cuh cov_spill_args.cuh"
DEPS[cov_mma]="common.cuh compat.cuh async_copy.cuh cov_spill_args.cuh mma_tf32.cuh"
DEPS[cgmm]="common.cuh compat.cuh hermitian_solve.cuh jacobi_coop.cuh"
DEPS[wpe]="common.cuh compat.cuh hermitian_solve.cuh jacobi_coop.cuh lu_coop.cuh auxiva.cuh"
DEPS[spatial]="common.cuh compat.cuh ssl.cuh"
DEPS[cm_mask]="common.cuh compat.cuh"
pids=()
for f in api generic weights weights_coop weights_post stft_cov_fused stft_cov_ws apply_istft_fused stft_spill cov_mma cgmm wpe spatial cm_mask; do
  stale=0
  [ -f "$OBJ/$f.o" ] || stale=1
  for d in "$f.cu" ${DEPS[$f]} ../../include/setk_b200.h build.sh; do
    [ "$HERE/$d" -nt "$OBJ/$f.o" ] && stale=1
  done
  if [ $stale -eq 1 ]; then
    ( $NVCC $FLAGS -Xptxas -v -c "$HERE/$f.cu" -o "$OBJ/$f.o.tmp" > "$OBJ/$f.log" 2>&1 && mv "$OBJ/$f.o.tmp" "$OBJ/$f.o" ) &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
if [ $rc -ne 0 ]; then cat "$OBJ"/*.log | grep -v "^ptxas info" | head -100; exit 1; fi
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT" "$OBJ"/api.o "$OBJ"/generic.o "$OBJ"/weights.o "$OBJ"/weights_coop.o "$OBJ"/weights_post.o "$OBJ"/stft_cov_fused.o "$OBJ"/stft_cov_ws.o "$OBJ"/apply_istft_fused.o "$OBJ"/stft_spill.o "$OBJ"/cov_mma.o "$OBJ"/cgmm.o "$OBJ"/wpe.o "$OBJ"/spatial.o "$OBJ"/cm_mask.o
echo "built $OUT"
