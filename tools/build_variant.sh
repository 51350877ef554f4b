#!/bin/bash
# tools/build_variant.sh NAME "-DDVA_RING_STAGES=4 ..." [file.cu ...]
# Rebuilds the given sources (default: view_attention_ring.cu) with extra defines and links a
# tuning variant build_variants/libdva_NAME.so from them plus the stock objects
# (load it with DVA_B200_LIB=build_variants/libdva_NAME.so).
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
NAME=$1; DEFS=$2; shift 2 || true
FILES=${@:-view_attention_ring.cu}
CS=$ROOT/deepviewagg_b200/csrc
OUT=$ROOT/build_variants; mkdir -p $OUT/obj_$NAME
OBJS=""
for f in $FILES; do
  o=$OUT/obj_$NAME/${f%.cu}.o
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr $DEFS -c $CS/$f -o $o
  OBJS="$OBJS $o"
done
STOCK=""
for o in $CS/build/*.o; do
  b=$(basename $o); skip=0
  for f in $FILES; do [ "$b" == "${f%.cu}.o" ] && skip=1; done
  [ $skip == 0 ] && STOCK="$STOCK $o"
done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $OUT/libdva_$NAME.so $OBJS $STOCK -lcudart
echo built $OUT/libdva_$NAME.so
