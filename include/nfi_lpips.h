/*
 * nfi_lpips.h -- C ABI of the LPIPS-VGG distance of the inversion loss (SURVEY.md section 8f, N4).
 *
 * Reference: lib/metrics.py:97-137 (LPIPSLoss over lpips.LPIPS(net='vgg')), the two-tensor form
 * every run.py call site uses:
 *
 *   x'  = (x - shift) / scale                                      ScalingLayer
 *   f_l = VGG16 features at relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 (13 3x3 convs, 4 max pools)
 *   n_l = f_l / (||f_l||_channels + 1e-10)                         normalize_tensor
 *   d   = sum_l mean_{h,w} sum_c lin_l[c] (n_l(in0) - n_l(in1))^2  NetLinLayer (1x1, no bias)
 *
 * in0 and in1 run through the network as one 2N-image batch.  conv1_1 (3 -> 64) runs in fp32 on
 * the CUDA cores; the other twelve convs on the synthesis network's TMA / wgmma kernel with bf16
 * hi / lo pair operands (README design 4.6, 4.8).  The per-image distance is summed in a fixed order
 * without cross-image atomics: an image's distance and gradient do not depend on the batch around
 * it.
 *
 * Conventions as in nfi_render.h: device pointers, fp32, stream as void*, 0 = success.
 */
#ifndef NFI_LPIPS_H_
#define NFI_LPIPS_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_LPIPS_CONVS 13 /* conv1_1 .. conv5_3 */
#define NFI_LPIPS_TAPS 5   /* relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 */

typedef struct nfi_lpips_params {
  int32_t n;      /* N image pairs (> 0) */
  int32_t height; /* H, a multiple of 16 (four 2x2 pools) */
  int32_t width;  /* W, a multiple of 16 */
  int32_t save;   /* 0: distance only; 1: the forward keeps what nfi_lpips_backward reads for a
                     gradient to in0; 2: also room for a gradient to in1 (larger workspaces) */
  const float *in0; /* [N,3,H,W] */
  const float *in1; /* [N,3,H,W] */
  const float *conv_w[NFI_LPIPS_CONVS]; /* [Cout,Cin,3,3] */
  const float *conv_b[NFI_LPIPS_CONVS]; /* [Cout] */
  const float *lin_w[NFI_LPIPS_TAPS];   /* [C] of the tap (64, 128, 256, 512, 512) */
  const float *shift; /* [3] */
  const float *scale; /* [3] */
  float *out;         /* [N] distance */
  void *workspace;
  size_t workspace_bytes;
} nfi_lpips_params;

/* Workspace of a forward with params->save as given (0 on invalid sizes). */
NFI_API size_t nfi_lpips_workspace_bytes(const nfi_lpips_params *params);
NFI_API int nfi_lpips_forward(const nfi_lpips_params *params, void *stream);
/* After a forward with save = 1 or 2 on the same params and workspace: grad_in0 [N,3,H,W] +=
 * d(sum_i g_dist[i] out[i]) / d in0, and, if grad_in1 is not NULL (save = 2 only), grad_in1 +=
 * the same for in1.  Where a tap's feature vector is entirely zero the gradient through its
 * normalisation is 0 (the reference's autograd gives NaN there). */
NFI_API int nfi_lpips_backward(const nfi_lpips_params *params, const float *g_dist, float *grad_in0,
                               float *grad_in1, void *stream);
/* After a forward with save = 1 or 2: copies conv `layer`'s (0 .. 12) pre-activation u [2N,h,w,Cout]
 * (channel-last, in0's images first) to out.  Its signs and window maxima are the ReLU and pool
 * branches the backward takes (tests compare against float64 on those branches). */
NFI_API int nfi_lpips_saved_preactivation(const nfi_lpips_params *params, int32_t layer, float *out,
                                          void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_LPIPS_H_ */
