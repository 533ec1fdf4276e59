/*
 * nfi_disc.h -- C ABI of the GAN discriminator's backbone (the G step's D(fake) call and the D
 * step's D(real) / D(fake) calls; the R1 call stays with the module).
 *
 * Reference: models/stylegan.py:493-676 (DiscriminatorBackbone.forward after the conditioning
 * vector; cmap is the mapping network's output and enters as an input).  With R the image side and
 * C(r) = min(32768 / r, 512) the channels at resolution r, the blocks run at r = R, R/2, .., 8:
 *
 *   x      = lrelu(sqrt2 (fromrgb(img) + b))                    (block R only; 1x1, nc -> C(R))
 *   skip   = sqrt2/2 conv1x1(downsample2d(x))                   4x4 [1,3,3,1] FIR, stride 2, pad 1
 *   a      = lrelu(sqrt2 (conv0(x) + b0))                       3x3, pad 1, C(r) -> C(r)
 *   x'     = lrelu(conv1(filter2d^T(a)) + b1) + skip            FIR pad 1, 3x3 stride 2, -> C(r/2)
 *
 * then at 4x4 (512 channels): minibatch std over groups of 4 (images b, b + B/4, b + B/2,
 * b + 3B/4), conv 3x3 513 -> 512 + lrelu sqrt2, fc 8192 -> 512 + lrelu sqrt2, out 512 -> N (N =
 * cmap_dim, or 1 without conditioning), logits = sum(out * cmap) / sqrt(cmap_dim) (or out).
 * Every lrelu has slope 0.2, every weight its equalized-lr gain.
 *
 * The 3x3 and 1x1 convs of the blocks run on the synthesis network's TMA / wgmma kernel with
 * bf16 hi / lo pair operands (README design 4.6, 4.10), their weight gradients on its
 * weight-gradient kernel; fromrgb and the 4x4 epilogue run in fp32 on the CUDA cores.  Every sum
 * over positions or images has a fixed order and there are no cross-image atomics.
 *
 * Conventions as in nfi_render.h: device pointers, fp32, stream as void*, 0 = success.
 */
#ifndef NFI_DISC_H_
#define NFI_DISC_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_DISC_MAX_BLOCKS 6 /* resolution blocks R .. 8 for R <= 256 */

typedef struct nfi_disc_params {
  int32_t batch;        /* B > 0, a multiple of 4 (the minibatch-std group) */
  int32_t resolution;   /* R: a power of two in 8..256 */
  int32_t img_channels; /* nc: 1..4 */
  int32_t cmap_dim;     /* 0 (unconditional: out has one channel) or 512 */
  int32_t save;         /* 1: the forward keeps what nfi_disc_backward reads */
  const float *img;     /* [B,nc,R,R] */
  const float *cmap;    /* [B,cmap_dim], NULL with cmap_dim 0 */
  const float *fromrgb_w; /* [C(R),nc,1,1] */
  const float *fromrgb_b; /* [C(R)] */
  /* block i at resolution R >> i (i < log2(R) - 2; the rest NULL) */
  const float *conv0_w[NFI_DISC_MAX_BLOCKS]; /* [C,C,3,3] */
  const float *conv0_b[NFI_DISC_MAX_BLOCKS]; /* [C] */
  const float *conv1_w[NFI_DISC_MAX_BLOCKS]; /* [C',C,3,3] (C' = C(r/2)) */
  const float *conv1_b[NFI_DISC_MAX_BLOCKS]; /* [C'] */
  const float *skip_w[NFI_DISC_MAX_BLOCKS];  /* [C',C,1,1] */
  const float *b4_conv_w; /* [512,513,3,3] */
  const float *b4_conv_b; /* [512] */
  const float *fc_w;      /* [512,8192] */
  const float *fc_b;      /* [512] */
  const float *out_w;     /* [N,512] */
  const float *out_b;     /* [N] */
  float *logits;          /* [B] */
  void *workspace;
  size_t workspace_bytes;
} nfi_disc_params;

/* Gradient outputs of nfi_disc_backward, each accumulated into (+=) and each optional (NULL: not
 * computed), laid out as the parameters above. */
typedef struct nfi_disc_grads {
  float *fromrgb_w;
  float *fromrgb_b;
  float *conv0_w[NFI_DISC_MAX_BLOCKS];
  float *conv0_b[NFI_DISC_MAX_BLOCKS];
  float *conv1_w[NFI_DISC_MAX_BLOCKS];
  float *conv1_b[NFI_DISC_MAX_BLOCKS];
  float *skip_w[NFI_DISC_MAX_BLOCKS];
  float *b4_conv_w;
  float *b4_conv_b;
  float *fc_w;
  float *fc_b;
  float *out_w;
  float *out_b;
} nfi_disc_grads;

/* Workspace of a forward with params->save as given (0 on invalid sizes). */
NFI_API size_t nfi_disc_workspace_bytes(const nfi_disc_params *params);
NFI_API int nfi_disc_forward(const nfi_disc_params *params, void *stream);
/* After a forward with save = 1 on the same params and workspace: the gradients of
 * sum(g_logits * logits) (g_logits [B]), accumulated into grad_img [B,nc,R,R] and grad_cmap
 * [B,cmap_dim] (each optional) and into the parameter gradients of `grads`. */
NFI_API int nfi_disc_backward(const nfi_disc_params *params, const float *g_logits, float *grad_img,
                              float *grad_cmap, const nfi_disc_grads *grads, void *stream);
/* After a forward with save = 1: copies a saved pre-activation (or an activation of the same
 * sign), fp32, to out.  Block i < log2(R) - 2: which 0 the fromrgb output [B,R,R,C] (block 0 only),
 * 1 the conv0 output [B,r,r,C], 2 the conv1 pre-activation [B,r/2,r/2,C'], channel-last.  Block
 * log2(R) - 2 (the 4x4 epilogue): which 0 the conv pre-activation [B,512,4,4], 1 the fc
 * pre-activation [B,512].  Where a value is positive the backward took the lrelu's unit-slope
 * branch (tests compare against float64 on those branches). */
NFI_API int nfi_disc_saved_preactivation(const nfi_disc_params *params, int32_t block, int32_t which,
                                         float *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_DISC_H_ */
