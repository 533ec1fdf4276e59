#!/bin/bash
# usage: bash tools/build_variant.sh <name> [-DNFI_... flags]
# Builds csrc/libnfi_render_<name>.so: the pipelined-kernel translation unit recompiled with the
# given macros, linked with the objects of the regular build (run csrc/build.sh first).  The
# variants are timed against the regular build on one box through NFI_LIB_PATH
# (tools/ab_forward.py, tools/time_backward.py).  Register / spill report: csrc/ptxas_<name>.txt.
set -e
name=$1; shift
cd "$(dirname "$0")/../nerf_from_image_b200/csrc"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 --fmad=false -lineinfo -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I../../include -Xptxas -v"
$NVCC $FLAGS -c -o nfi_pipe_$name.o nfi_pipe.cu "$@" 2> ptxas_$name.txt
$NVCC -shared -cudart static -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -o libnfi_render_$name.so nfi_render.o nfi_pipe_$name.o nfi_field.o nfi_synth.o nfi_heads.o nfi_viewdir.o
grep -A1 "render_forward_pipeILi12ELi0ELb1ELi3ELb0ELi2E\|render_backward_pipeILi12ELi0ELb[01]ELi2E" ptxas_$name.txt | grep -v "^--" | cut -c1-200
