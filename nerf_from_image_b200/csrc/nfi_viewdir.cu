// Translation unit of the view-direction-conditioned SIMT render (--use_viewdir, the CARLA
// models: run.py:216-217, models/generator.py:189-253,376-377,662-663): the launchers of
// render_forward_simt / render_backward_simt instantiated with VD = true, a unit of its own that
// build.sh compiles in parallel with the others.
#include "nfi_backward.cuh"

namespace nfi {
template int launch_forward_simt<true>(const nfi_render_params&, bool, cudaStream_t);
template int launch_backward_simt<true>(const nfi_render_params&, const nfi_render_grads&,
                                        cudaStream_t);
}  // namespace nfi
