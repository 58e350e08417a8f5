#!/bin/bash
# Builds tts_b200/libtts_b200.so (sm_90a only) in-tree.  Called by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p ../../build/obj
objs=""
newest_hdr=$(ls -t *.cuh ../../include/tts_b200.h | head -1)     # any header newer than an object rebuilds it
for f in *.cu; do
  o=../../build/obj/${f%.cu}.o
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ "$newest_hdr" -nt "$o" ]; then
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c "$f" -o "$o" &
  fi
  objs="$objs $o"
done
wait
$NVCC -shared --cudart static -o ../libtts_b200.so $objs
echo "built $(cd .. && pwd)/libtts_b200.so"
