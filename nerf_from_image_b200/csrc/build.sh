#!/bin/bash
# Builds libnfi_render.so in-tree for sm_90a (cross-compiles without a GPU).
# Nine translation units compiled in parallel: the pipelined tensor-core kernels (nfi_pipe.cu) and
# their view-direction-conditioned instantiations (nfi_pipe_vd.cu), both on the launchers of
# nfi_pipe_ladder.cuh; the sampler seam and pose kernels (nfi_field.cu), the synthesis network
# (nfi_synth.cu), the LPIPS-VGG loss and the encoder's regression heads on the synthesis network's
# conv kernels (nfi_lpips.cu, nfi_encoder.cu), the regulariser-head point evaluator (nfi_heads.cu),
# the view-direction-conditioned instantiations of the SIMT launchers (nfi_viewdir.cu), and everything else
# (nfi_render.cu: C ABI and routing, re-layout, plain SIMT kernels, stand-alone decoder).  Each
# kernel is compiled only in the unit that launches it.  nfi_render.cu and nfi_viewdir.cu take
# --split-compile 0 (their many kernels are optimised in parallel).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 --fmad=false -lineinfo -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I../../include ${NFI_PTXAS_V:+-Xptxas -v}"
$NVCC $FLAGS -c -o nfi_pipe.o nfi_pipe.cu "$@" &
pipe_pid=$!
$NVCC $FLAGS -c -o nfi_pipe_vd.o nfi_pipe_vd.cu "$@" &
pipe_vd_pid=$!
$NVCC $FLAGS -c -o nfi_field.o nfi_field.cu "$@" &
field_pid=$!
$NVCC $FLAGS -c -o nfi_synth.o nfi_synth.cu "$@" &
synth_pid=$!
$NVCC $FLAGS -c -o nfi_heads.o nfi_heads.cu "$@" &
heads_pid=$!
$NVCC $FLAGS -c -o nfi_lpips.o nfi_lpips.cu "$@" &
lpips_pid=$!
$NVCC $FLAGS -c -o nfi_encoder.o nfi_encoder.cu "$@" &
encoder_pid=$!
$NVCC $FLAGS --split-compile 0 -c -o nfi_viewdir.o nfi_viewdir.cu "$@" &
viewdir_pid=$!
$NVCC $FLAGS --split-compile 0 -c -o nfi_render.o nfi_render.cu "$@"
wait $pipe_pid
wait $pipe_vd_pid
wait $field_pid
wait $synth_pid
wait $heads_pid
wait $lpips_pid
wait $encoder_pid
wait $viewdir_pid
$NVCC -shared -cudart static -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -o libnfi_render.so nfi_render.o nfi_pipe.o nfi_pipe_vd.o nfi_field.o nfi_synth.o nfi_lpips.o nfi_encoder.o nfi_heads.o nfi_viewdir.o
