#!/bin/bash
# Builds libb200z.so in-tree for sm_90a (nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -diag-suppress 550"
mkdir -p _build
pids=()
objs=()
for src in *.cu; do
  f=${src%.cu}
  objs+=(_build/$f.o)
  stale=0
  [ -f _build/$f.o ] || stale=1
  for dep in $f.cu *.cuh ../../include/b200z.h build.sh; do
    [ $stale -eq 0 ] && [ $dep -nt _build/$f.o ] && stale=1
  done
  if [ $stale -eq 1 ]; then
    rm -f _build/$f.o # a failed compile must not leave an older object for the link step
    $NVCC $FLAGS -c $f.cu -o _build/$f.o &
    pids+=($!)
  fi
done
for pid in "${pids[@]}"; do
  wait "$pid" || { echo "build.sh: a compile failed" >&2; exit 1; }
done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../libb200z.so "${objs[@]}"
echo built ../libb200z.so
