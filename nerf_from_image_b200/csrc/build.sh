#!/bin/bash
# Builds libnfi_render.so in-tree for sm_90a (cross-compiles without a GPU).  Every nfi_*.cu here is
# one translation unit; they compile in parallel and the library links them all.  Each kernel is
# compiled only in the unit that launches it.  nfi_render.cu and nfi_viewdir.cu take
# --split-compile 0 (their many kernels are optimised in parallel).
#
#   build.sh [unit ...] [-nvcc-flag ...]
# With unit names (synth for nfi_synth.cu, ...) only those units are recompiled before the link;
# arguments that start with '-' go to every compile.  NFI_VARIANT=<name> compiles the named units
# to nfi_<unit>_<name>.o instead and links them with the other units' regular objects into
# libnfi_render_<name>.so (tools/build_variant.sh).  NFI_PTXAS_V=1 adds the register / spill report.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 --fmad=false -lineinfo -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I../../include ${NFI_PTXAS_V:+-Xptxas -v}"
all=()
for f in nfi_*.cu; do u=${f#nfi_}; all+=("${u%.cu}"); done
units=() flags=()
for a in "$@"; do
  case $a in
    -*) flags+=("$a") ;;
    *) [ -f "nfi_$a.cu" ] || { echo "build.sh: no unit nfi_$a.cu" >&2; exit 1; }; units+=("$a") ;;
  esac
done
[ ${#units[@]} -gt 0 ] || units=("${all[@]}")
obj() {  # the object of unit $1 that this build links
  case " ${units[*]} " in *" $1 "*) echo "nfi_$1${NFI_VARIANT:+_$NFI_VARIANT}.o" ;; *) echo "nfi_$1.o" ;; esac
}
pids=()
for u in "${units[@]}"; do
  split=()
  case $u in render|viewdir) split=(--split-compile 0) ;; esac
  $NVCC $FLAGS "${split[@]}" -c -o "$(obj "$u")" "nfi_$u.cu" "${flags[@]}" &
  pids+=($!)
done
failed=0
for p in "${pids[@]}"; do wait "$p" || failed=1; done
[ $failed = 0 ]
objs=()
for u in "${all[@]}"; do objs+=("$(obj "$u")"); done
$NVCC -shared -cudart static -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -o "libnfi_render${NFI_VARIANT:+_$NFI_VARIANT}.so" "${objs[@]}"
