#!/bin/bash
# tools/build_variant.sh NAME "-DSHINE_X=1 ..."  -> tools/variants/libshine_b200_NAME.so  (A/B runs: SHINE_B200_LIB=<path>)
set -e
cd "$(dirname "$0")/.."
NAME=$1; shift
OBJS=""
mkdir -p tools/variants
for f in shine_mapping_b200/csrc/*.cu; do
  o=/tmp/variant_${NAME}_$(basename ${f%.cu}).o
  nvcc "$@" -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I include -I shine_mapping_b200/csrc -c -o $o $f &
  OBJS="$OBJS $o"
done
wait
nvcc -gencode arch=compute_90a,code=sm_90a --shared -Xcompiler -fPIC -o tools/variants/libshine_b200_${NAME}.so $OBJS
echo built tools/variants/libshine_b200_${NAME}.so
