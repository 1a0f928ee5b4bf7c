#!/bin/bash
# Development helper: build a variant of the library.
#   tools/build_variant.sh NAME [--base DIR] FILE.cu[:"-DFOO=1 ..."] ...   ->  zstd_b200/variants/libzstd_b200_NAME.so
# The listed files are compiled (with their extra flags); every other object comes from DIR (objects of another build, e.g.
# the previous commit's) when --base is given, else from the current build.  Select a variant at run time with
# ZSTDB200_LIB=<path> (tests/variant_sweep.py, tests/wave_sweep.py, tests/profile_one.py).
set -e
cd "$(dirname "$0")/../zstd_b200/csrc"
name=$1; shift
base=.
if [ "$1" == "--base" ]; then base=$2; shift 2; fi
mkdir -p ../variants /tmp/zbv_$name
[ "$base" == "." ] && make -s all
declare -A flags
for spec in "$@"; do f=${spec%%:*}; fl=""; [[ "$spec" == *:* ]] && fl=${spec#*:}; flags[$f]="x$fl"; done
objs=""
for f in zb_api zb_dict zb_match zb_ldm zb_seqimport zb_literals zb_sequences zb_stitch zb_decode; do
  if [ -n "${flags[$f.cu]}" ]; then
    nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fvisibility=hidden -Xptxas -v ${flags[$f.cu]#x} -c $f.cu -o /tmp/zbv_$name/$f.o 2> /tmp/zbv_$name/$f.log
    grep "spill" /tmp/zbv_$name/$f.log | grep -v " 0 bytes spill stores, 0 bytes spill loads" | head -4 || true
    objs="$objs /tmp/zbv_$name/$f.o"
  else objs="$objs $base/$f.o"; fi
done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../variants/libzstd_b200_$name.so $objs -lcudart
echo built ../variants/libzstd_b200_$name.so
