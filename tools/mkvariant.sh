#!/bin/bash
# tools/mkvariant.sh NAME "EXTRA_NVCC_FLAGS" file1.cu [file2.cu ...]
# Build variants/NAME.so: the listed kernels recompiled with the extra flags (usually -D tuning macros), everything else
# taken from the regular build (vello_b200/csrc/build/*.o must be up to date: run make first). For tools/variant_check.py / ab.sh.
set -e
name=$1; extra=$2; shift 2
cd "$(dirname "$0")/../vello_b200/csrc"
mkdir -p ../../variants /tmp/mkvariant_$name
objs=""
for o in build/*.o; do
  b=$(basename $o .o); skip=0
  for f in "$@"; do [ "$b.cu" == "$f" ] && skip=1; done
  [ $skip == 0 ] && objs="$objs $o"
done
for f in "$@"; do
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false -Xcompiler -fPIC $extra -c $f -o /tmp/mkvariant_$name/${f%.cu}.o &
done
wait
for f in "$@"; do objs="$objs /tmp/mkvariant_$name/${f%.cu}.o"; done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../variants/$name.so $objs
echo built variants/$name.so
