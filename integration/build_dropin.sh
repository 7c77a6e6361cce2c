#!/bin/bash
# Builds the reference's own drivers (main.cpp -> ntt-b200, RS.cpp -> rs-b200) UNMODIFIED against the H100 library.
# Needs the reference tree (default /root/reference); outputs go to oracle/_ref/dropin/ (git-ignored, travels to
# the GPU box with gpurun).  Nothing from the reference is copied: the staging directory only holds symlinks.
set -euo pipefail
REF=${REF:-/root/reference}
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT="$ROOT/oracle/_ref/dropin"
[ -f "$REF/ntt.cpp" ] || { echo "reference tree $REF not present: keeping prebuilt $OUT (if any)"; exit 0; }
python "$ROOT/fastecc_b200/build.py" >/dev/null
rm -rf "$OUT/stage"; mkdir -p "$OUT/stage"
for f in main.cpp RS.cpp "GF(p).cpp" SIMD.h LargePages.cpp wall_clock_timer.h; do ln -s "$REF/$f" "$OUT/stage/$f"; done
ln -s "$ROOT/fastecc_b200/shim/ntt.cpp" "$OUT/stage/ntt.cpp"          # <- the only substitution
FLAGS=(-std=c++1y -O3 -fopenmp -mavx2 -DSIMD=AVX2 "-DFASTECC_REF_NTT_CPP=\"$REF/ntt.cpp\"" -I"$ROOT/include")
LIBS=(-L"$ROOT/fastecc_b200" -lfastecc_b200 -Wl,-rpath,'$ORIGIN/../../../fastecc_b200')
/usr/bin/g++ "${FLAGS[@]}" -o "$OUT/rs-b200"  "$OUT/stage/RS.cpp"   "${LIBS[@]}"
/usr/bin/g++ "${FLAGS[@]}" -o "$OUT/ntt-b200" "$OUT/stage/main.cpp" "${LIBS[@]}"
echo "built $OUT/rs-b200 $OUT/ntt-b200"
