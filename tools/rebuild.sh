#!/bin/bash
# Recompiles only the named translation units (pipe pipe_vd render field synth heads viewdir) and relinks.
# usage: bash tools/rebuild.sh pipe [render ...]
cd "$(dirname "$0")/../nerf_from_image_b200/csrc" || exit 1
FLAGS="-O3 -std=c++17 --fmad=false -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I../../include"
pids=()
for tu in "$@"; do
  extra=""
  case $tu in render|viewdir) extra="--split-compile 0";; esac
  ( nvcc $FLAGS $extra ${NFI_PTXAS_V:+-Xptxas -v} -c -o nfi_$tu.o nfi_$tu.cu 2>&1 | grep -E "error|warning|${NFI_GREP:-zzzz}" -A3 | head -40 ) &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
nvcc -shared -cudart static -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -o libnfi_render.so \
  nfi_render.o nfi_pipe.o nfi_pipe_vd.o nfi_field.o nfi_synth.o nfi_heads.o nfi_viewdir.o && ls -la libnfi_render.so
