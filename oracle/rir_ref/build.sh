#!/bin/bash
# Compile the reference's own image-method generator (include/rir-generator.cc, what its
# rir-simulate runs) against the stand-in headers here, into oracle/_ref/rir_ref.  Nothing from
# the reference is copied: the driver includes its source by path.  Skipped (exit 0) when the
# reference tree is absent.  TEST INFRASTRUCTURE ONLY.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${SETK_REFERENCE:-/root/reference}"
OUT="$HERE/../_ref/rir_ref"
if [ ! -f "$REF/include/rir-generator.cc" ]; then
  echo "rir_ref: no reference tree at $REF, skipped"
  exit 0
fi
mkdir -p "$(dirname "$OUT")"
${CXX:-g++} -O2 -std=c++17 -I"$HERE" -I"$REF" "-DRIR_GENERATOR_CC=\"$REF/include/rir-generator.cc\"" \
  "$HERE/rir_ref_main.cc" -o "$OUT.tmp"
mv "$OUT.tmp" "$OUT"
echo "built $OUT"
