#!/bin/bash
# Build the CPU-emulated twin of libsetk_b200.so for the CPU test tier.
# TEST INFRASTRUCTURE ONLY: the product never loads this library.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
SRC="$ROOT/setk_b200/csrc"
OUT="$HERE/libsetk_b200_emu.so"
OBJ="$HERE/obj"
mkdir -p "$OBJ"
pids=()
objs=("$OBJ/cuda_emu.o")
for src in "$SRC"/*.cu; do
  o="$OBJ/$(basename "$src" .cu).o"
  objs+=("$o")
  g++ -O2 -std=c++17 -DSETK_EMU -DSETK_TABLE_CHUNK=8 -fPIC -pthread -I"$HERE" -I"$ROOT/include" -x c++ -c "$src" -o "$o" &
  pids+=($!)
done
g++ -O2 -std=c++17 -DSETK_EMU -fPIC -pthread -I"$HERE" -c "$HERE/cuda_emu.cc" -o "$OBJ/cuda_emu.o" &
pids+=($!)
for p in "${pids[@]}"; do wait $p; done
g++ -shared -pthread -o "$OUT" "${objs[@]}"
echo "built $OUT"
