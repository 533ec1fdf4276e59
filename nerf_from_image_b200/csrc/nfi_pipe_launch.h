// Launchers of the pipelined tensor-core kernels.  VD: the view-direction-conditioned decoder
// (params.view_features / w3 / b3, w2 of 33 rows).  The ladders are templates
// (nfi_pipe_ladder.cuh); nfi_pipe.cu instantiates them for VD = false and nfi_pipe_vd.cu for
// VD = true, two units that build.sh compiles in parallel with the rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_render.h"

namespace nfi {
// the weight image at `wimg` (nfi_layout.h: its workspace slot), then render_forward_pipe on
// `grid` persistent CTAs; `scratch` = pipe_scratch_bytes_per_cta per CTA
template <bool VD>
int launch_pipe_forward(const nfi_render_params& p, unsigned char* wimg, float* scratch,
                        unsigned grid, cudaStream_t st);
size_t pipe_scratch_bytes_per_cta(int num_samples, int nes);
// both weight images at `wimg` (nfi_layout.h), then render_backward_pipe: a frozen decoder (and
// with a view a frozen mapper output); decoder gradients of `g` are not produced
template <bool VD>
int launch_pipe_backward(const nfi_render_params& p, const nfi_render_grads& g,
                         unsigned char* wimg, unsigned grid, cudaStream_t st);
// decoder-weight gradients (grad_w1 / b1 / w2 / b2 of `g`, accumulated) on the tensor cores: both
// weight images + render_wgrad_pipe, whose accumulator rows follow them (nfi_layout.h,
// NFI_BACKWARD_WORKSPACE_BYTES in all).  The other gradients of `g` are produced only with
// `planes`: ONE sweep for the whole generator step, grad_planes / grad_palette / grad_beta /
// grad_alpha (no pose gradient).
int launch_pipe_wgrad(const nfi_render_params& p, const nfi_render_grads& g, unsigned char* wimg,
                      unsigned grid, bool planes, cudaStream_t st);
// composited surface normals (params.normals, overwritten) after a render_forward_pipe launch of
// the same params (z_fine and mask filled): render_normals_pipe, reading the plain weight image
// at `wimg` (rebuilt there after a view render) and a backward image it builds at `wimg_bwd`
int launch_pipe_normals(const nfi_render_params& p, unsigned char* wimg, unsigned char* wimg_bwd,
                        unsigned grid, cudaStream_t st);
}  // namespace nfi
