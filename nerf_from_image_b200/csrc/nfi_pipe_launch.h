// Launchers of the pipelined tensor-core kernels (nfi_pipe.cu), a translation unit of its own so
// that build.sh can compile it in parallel with the rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_render.h"

namespace nfi {
// render_forward_pipe for (nout_pad, extra_mode, fine_sampling, S, debug bits of mlp_mode) on
// `grid` persistent CTAs; `wimg` = weight image (prep_weight_image with the pipelined
// kernel's scalings), `scratch` = pipe_scratch_floats(S, nes) floats per CTA.
int launch_pipe_forward(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                        float* scratch, unsigned grid, cudaStream_t st, char* err, size_t err_len);
// both weight images (64 KiB at `wimg`) + render_backward_pipe
int launch_pipe_backward(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                         unsigned char* wimg, unsigned grid, cudaStream_t st, char* err,
                         size_t err_len);
// decoder-weight gradients (grad_w1 / b1 / w2 / b2 of `g`, accumulated) on the tensor cores: both weight
// images + render_wgrad_pipe; the other gradients of `g` are NOT produced (launch_pipe_backward)
// (workspace at `wimg`: the two weight images, then one accumulator row buffer per CTA:
// pipe_wgrad_workspace_bytes(grid) in all)
size_t pipe_wgrad_workspace_bytes(unsigned grid);
// `planes`: ONE sweep for the whole generator step -- the kernel also produces grad_planes /
// grad_palette / grad_beta / grad_alpha of `g` (no pose gradient)
int launch_pipe_wgrad(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                      unsigned char* wimg, unsigned grid, bool planes, cudaStream_t st, char* err,
                      size_t err_len);
// composited surface normals (params.normals, overwritten) after a render_forward_pipe launch of
// the same params (z_fine and mask filled): render_normals_pipe
int launch_pipe_normals(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                        unsigned char* wimg_bwd, unsigned grid, cudaStream_t st, char* err,
                        size_t err_len);
// the pipelined kernels' weight image (log2 e folded into layer 1 and the colour rows of
// layer 2, padded logits at -1e30)
int launch_pipe_weight_image(const nfi_render_params& p, unsigned char* wimg, cudaStream_t st);
size_t pipe_scratch_bytes_per_cta(int num_samples, int nes);
// The view-direction-conditioned render (params.view_features / w3 / b3, w2 of 33 rows) on
// render_forward_pipe<..., VD = true> (nfi_pipe_vd.cu): its weight image (nfi_layout.h, up to
// 64 KiB at `wimg`) and the launch, `scratch` and `grid` as for launch_pipe_forward.
int launch_pipe_weight_image_vd(const nfi_render_params& p, unsigned char* wimg, cudaStream_t st);
int launch_pipe_forward_vd(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                           float* scratch, unsigned grid, cudaStream_t st, char* err,
                           size_t err_len);
// Its backward with a frozen decoder and mapper output (no grad_w1 .. grad_b3):
// render_backward_pipe<..., VD = true> and both weight images (kVdBackwardWorkspaceBytes at
// `wimg`, nfi_layout.h).
int launch_pipe_backward_vd(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                            unsigned char* wimg, unsigned grid, cudaStream_t st, char* err,
                            size_t err_len);
}  // namespace nfi
