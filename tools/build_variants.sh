#!/bin/bash
# usage: tools/build_variants.sh name1 "flags1" name2 "flags2" ...  -> tools/variants/lib_<name>.so
cd "$(dirname "$0")/.."
mkdir -p tools/variants
while [ $# -gt 1 ]; do
  name=$1; flags=$2; shift 2
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared $flags \
    -o tools/variants/lib_$name.so ddsp_b200/csrc/capi.cu &
done
wait
ls -la tools/variants/
