#!/bin/bash
# Recompiles only the named translation units (synth for nfi_synth.cu, ...) and relinks.
# usage: bash tools/rebuild.sh pipe [render ...]
exec bash "$(dirname "$0")/../nerf_from_image_b200/csrc/build.sh" "$@"
