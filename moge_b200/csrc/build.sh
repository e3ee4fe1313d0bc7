#!/bin/bash
# Build libmoge_b200.so for sm_90a (H100), in-tree: moge_b200/_lib/libmoge_b200.so.
set -e
cd "$(dirname "$0")"
OUT=../_lib
# MG_VARIANT=name builds an A/B variant next to the product library: objects in build_name/, _lib/libmoge_b200_name.so
# (selected at run time with MOGE_B200_LIB=<path>; tools/ab_variants.py)
BUILD=build${MG_VARIANT:+_$MG_VARIANT}
LIB=libmoge_b200${MG_VARIANT:+_$MG_VARIANT}.so
mkdir -p $OUT $BUILD
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I../../include $MG_EXTRA_FLAGS"
# a change of flags (e.g. MG_EXTRA_FLAGS=-DMG_ATT_DEBUG) invalidates every object
if [ "$(cat $BUILD/.flags 2>/dev/null)" != "$FLAGS" ]; then rm -f $BUILD/*.o; echo "$FLAGS" > $BUILD/.flags; fi
pids=()
for f in gemm_rows gemm_tiles conv64 convh gemm attention elementwise pack tmap peer engine; do
  if [ ! -f $BUILD/$f.o ] || [ $f.cu -nt $BUILD/$f.o ] || [ -n "$(find . -maxdepth 1 \( -name '*.cuh' -o -name '*.h' \) -newer $BUILD/$f.o)" ] || [ ../../include/moge_b200.h -nt $BUILD/$f.o ]; then
    ( nvcc $FLAGS -Xptxas -v -c $f.cu -o $BUILD/$f.o > $BUILD/$f.log 2>&1 || { echo "FAILED $f"; grep -E "error" $BUILD/$f.log | head -20; exit 1; } ) &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
[ $rc -eq 0 ] || exit 1
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $OUT/$LIB $BUILD/*.o -lcudart
echo "built $OUT/$LIB"
