#!/bin/bash
# usage: bash tools/build_variant.sh <name> [-DNFI_... flags]
# Builds csrc/libnfi_render_<name>.so: the pipelined-kernel translation unit recompiled with the
# given macros, linked with the objects of the regular build (run csrc/build.sh first).  The
# variants are timed against the regular build on one box through NFI_LIB_PATH
# (tools/ab_forward.py, tools/time_backward.py).  Register / spill report: csrc/ptxas_<name>.txt.
set -e
name=$1; shift
csrc="$(dirname "$0")/../nerf_from_image_b200/csrc"
NFI_VARIANT=$name NFI_PTXAS_V=1 bash "$csrc/build.sh" pipe "$@" 2> "$csrc/ptxas_$name.txt"
grep -A1 "render_forward_pipeILi12ELi0ELb1ELi3ELb0ELi2E\|render_backward_pipeILi12ELi0ELb[01]ELi2E" "$csrc/ptxas_$name.txt" |
  grep -v "^--" | cut -c1-200
