/*
 * nfi_encoder.h -- C ABI of the bootstrap encoder's regression heads (encoder training,
 * train_coord_regressor; SURVEY.md section 8f).
 *
 * Reference: models/encoder.py:70-103 (BootstrapEncoder.forward) from the backbone output(s) on:
 *
 *   x0     = relu(interpolate(features, x4, bilinear, align_corners=False))   [B,C,4h,4w]
 *   a1     = relu(post[0](x0)),  a2 = relu(post[2](a1))                       3x3, pad 1, C -> C
 *   maps   = post[4](a2)                                                      3x3, pad 1, C -> 4
 *   xl     = relu(features_latent)                                            [B,C,h,w]
 *   pooled = mean_{y,x} relu(w_regressor_pre[0](xl))                          3x3, pad 1, C -> C
 *
 * The backbones, w_regressor_post, the sigmoid of the mask channel and the losses stay with the
 * caller.  The five convs run on the synthesis network's TMA / wgmma kernel with bf16 hi / lo pair
 * operands (README design 4.6, 4.9); their weight gradients on its weight-gradient kernel.  Every
 * sum over positions or images has a fixed order and there are no cross-image atomics: an image's
 * outputs do not depend on the batch around it, and two backward calls give the same bits.
 *
 * Conventions as in nfi_render.h: device pointers, fp32, stream as void*, 0 = success.
 */
#ifndef NFI_ENCODER_H_
#define NFI_ENCODER_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_ENCODER_MAPS 4 /* post[4]'s outputs: three coordinates and the mask logit */

typedef struct nfi_encoder_params {
  int32_t batch;            /* B > 0 */
  int32_t height;           /* h of the features (the image is 4h x 4w) */
  int32_t width;            /* w */
  int32_t channels;         /* C of the features and of every head conv but post[4]: a multiple of 64 */
  int32_t pose_regressor;   /* 1: the post head (maps) */
  int32_t latent_regressor; /* 1: the w_regressor_pre head (pooled) */
  int32_t save;             /* 1: the forward keeps what nfi_encoder_backward reads */
  const float *features;        /* [B,C,h,w] the backbone output (NULL without the pose head) */
  const float *features_latent; /* [B,C,h,w] the latent backbone's output; may be `features`;
                                   NULL without the latent head */
  const float *post0_w;  /* [C,C,3,3] */
  const float *post0_b;  /* [C] */
  const float *post2_w;  /* [C,C,3,3] */
  const float *post2_b;  /* [C] */
  const float *post4_w;  /* [4,C,3,3] */
  const float *post4_b;  /* [4] */
  const float *wpre_w;   /* [C,C,3,3] w_regressor_pre[0] */
  const float *wpre_b;   /* [C] */
  float *maps;           /* [B,4h,4w,4] post[4]'s output, channel-last */
  float *pooled;         /* [B,C] */
  void *workspace;
  size_t workspace_bytes;
} nfi_encoder_params;

/* Gradient outputs of nfi_encoder_backward, each accumulated into (+=) and each optional (NULL:
 * not computed).  g_features_latent may be the same buffer as g_features (one shared backbone). */
typedef struct nfi_encoder_grads {
  float *g_features;        /* [B,C,h,w] */
  float *g_features_latent; /* [B,C,h,w] */
  float *g_post0_w;
  float *g_post0_b;
  float *g_post2_w;
  float *g_post2_b;
  float *g_post4_w;
  float *g_post4_b;
  float *g_wpre_w;
  float *g_wpre_b;
} nfi_encoder_grads;

/* Workspace of a forward with params->save as given (0 on invalid sizes). */
NFI_API size_t nfi_encoder_workspace_bytes(const nfi_encoder_params *params);
NFI_API int nfi_encoder_forward(const nfi_encoder_params *params, void *stream);
/* After a forward with save = 1 on the same params and workspace: the gradients of
 * sum(g_maps * maps) + sum(g_pooled * pooled).  g_maps [B,4h,4w,4] is read with the pose head,
 * g_pooled [B,C] with the latent head. */
NFI_API int nfi_encoder_backward(const nfi_encoder_params *params, const float *g_maps,
                                 const float *g_pooled, const nfi_encoder_grads *grads, void *stream);
/* After a forward with save = 1: copies a saved post-ReLU activation, channel-last fp32, to out:
 * layer 0 x0 [B,4h,4w,C], 1 a1, 2 a2 (same shape), 3 xl [B,h,w,C], 4 relu(w_regressor_pre[0](xl))
 * [B,h,w,C].  Where a value is positive the backward took the ReLU's pass branch (tests compare
 * against float64 on those branches). */
NFI_API int nfi_encoder_saved_activation(const nfi_encoder_params *params, int32_t layer, float *out,
                                         void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_ENCODER_H_ */
