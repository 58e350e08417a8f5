#!/bin/bash
# Builds tts_b200/libtts_b200.so (sm_90a only) in-tree.  Called by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p ../../build/obj
objs=""
pids=(); pid_objs=()
newest_hdr=$(ls -t *.cuh ../../include/tts_b200.h | head -1)     # any header newer than an object rebuilds it
for f in *.cu; do
  o=../../build/obj/${f%.cu}.o
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ "$newest_hdr" -nt "$o" ]; then
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c "$f" -o "$o" &
    pids+=($!); pid_objs+=("$o")
  fi
  objs="$objs $o"
done
# a failed nvcc leaves the file's previous object behind: delete it and stop, so no link picks up the stale object
failed=0
for i in "${!pids[@]}"; do wait "${pids[$i]}" || { rm -f "${pid_objs[$i]}"; failed=1; }; done
[ "$failed" -eq 0 ] || { echo "build.sh: compile failed; not linking" >&2; exit 1; }
$NVCC -shared --cudart static -o ../libtts_b200.so $objs
echo "built $(cd .. && pwd)/libtts_b200.so"
