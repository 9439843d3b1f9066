#!/bin/bash
# usage: tools/build_variants.sh name1 "flags1" name2 "flags2" ...  -> tools/variants/lib_<name>.so
# Each variant is the library's build (ddsp_b200/build.py) with the extra nvcc flags.
set -e
cd "$(dirname "$0")/.."
mkdir -p tools/variants
while [ $# -gt 1 ]; do
  name=$1; flags=$2; shift 2
  python -c 'import sys; from ddsp_b200 import build; build.build(out=sys.argv[1], flags=sys.argv[2].split())' \
    "tools/variants/lib_$name.so" "$flags"
done
ls -la tools/variants/
