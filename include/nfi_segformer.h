/*
 * nfi_segformer.h -- C ABI of the bootstrap encoder's SegFormer-B5 backbone (encoder training,
 * train_coord_regressor; models/segformer.py:175-275, Segformer.forward).
 *
 * The module: four stages of widths 64 / 128 / 320 / 512, heads 1 / 2 / 5 / 8 (head dimension 64),
 * MLP ratio 4, spatial-reduction ratios 8 / 4 / 2 / 1, any depth >= 1 per stage; a decoder head of
 * width 768 (linear_c4 .. linear_c1, linear_fuse) and linear_pred to out_features channels.  Images
 * are square, H a multiple of 32 in 32..256, so every stage's attention has (H/32)^2 <= 64 keys.
 *
 * Token GEMMs run on the synthesis network's TMA / wgmma kernel with bf16 hi / lo pair operands
 * (README design 4.6, 4.11), the rest on the CUDA cores in fp32.  The decoder head runs linear_c_i
 * and linear_fuse's column slice i at stage i's resolution, then upsamples and sums (the bilinear
 * upsample commutes with a 1x1 layer).  Every sum has a fixed order and there are no atomics: an
 * image's features do not depend on the batch around it, and two backward calls give the same bits.
 *
 * Conventions as in nfi_render.h: device pointers, fp32, stream as void*, 0 = success.
 */
#ifndef NFI_SEGFORMER_H_
#define NFI_SEGFORMER_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_SEGFORMER_STAGES 4
#define NFI_SEGFORMER_MAX_DEPTH 64  /* blocks per stage */
#define NFI_SEGFORMER_DECODER 768   /* decoder_dim */

/*
 * `params` is a host array of device pointers in the module's named_parameters() order:
 *   patch_embed1 .. patch_embed4, each: proj.weight, proj.bias, norm.weight, norm.bias;
 *   then for each stage i = 1..4: each block of block<i>:
 *     norm1.weight, norm1.bias, attn.q.weight, attn.q.bias, attn.kv.weight, attn.kv.bias,
 *     attn.proj.weight, attn.proj.bias,
 *     attn.sr.weight, attn.sr.bias, attn.norm.weight, attn.norm.bias   (stages 1-3, sr > 1, only),
 *     norm2.weight, norm2.bias, mlp.fc1.weight, mlp.fc1.bias, mlp.dwconv.dwconv.weight,
 *     mlp.dwconv.dwconv.bias, mlp.fc2.weight, mlp.fc2.bias;
 *   and the stage's norm<i>.weight, norm<i>.bias;
 *   then linear_c4.proj, linear_c3.proj, linear_c2.proj, linear_c1.proj (weight, bias each),
 *   linear_fuse.weight, linear_fuse.bias, linear_pred.weight, linear_pred.bias.
 * That is 16 + 20 (d1 + d2 + d3) + 16 d4 + 8 + 12 tensors: 1,064 at B5's depths (3, 6, 40, 3).
 */
typedef struct nfi_segformer_params {
  int32_t batch;        /* B > 0 */
  int32_t height;       /* H of the image: a multiple of 32 in 32..256 */
  int32_t width;        /* W == H */
  int32_t depths[NFI_SEGFORMER_STAGES];  /* blocks per stage, 1..NFI_SEGFORMER_MAX_DEPTH */
  int32_t out_features; /* linear_pred's outputs: a positive multiple of 64 */
  int32_t save;         /* 1: the forward keeps what nfi_segformer_backward reads */
  const float *image;   /* [B,3,H,W] */
  const float *const *params;  /* host array, the order above */
  const float *drop_scales;    /* [2 * sum(depths), B]: row 2k scales block k's attention branch,
                                  row 2k + 1 its MLP branch (blocks counted across the stages);
                                  the drop-path draws divided by keep_p, 1 where a block draws
                                  nothing.  NULL: all 1 (eval mode) */
  float *features;      /* [B,out_features,H/4,W/4] */
  void *workspace;
  size_t workspace_bytes;
} nfi_segformer_params;

/* Workspace of a forward with params->save as given (0 on invalid sizes). */
NFI_API size_t nfi_segformer_workspace_bytes(const nfi_segformer_params *params);
NFI_API int nfi_segformer_forward(const nfi_segformer_params *params, void *stream);
/* After a forward with save = 1 on the same params and workspace: the gradients of
 * sum(g_features * features) to the parameters.  `grads` is a host array parallel to params->params;
 * each entry is optional (NULL: not computed) and is accumulated into (+=).  There is no image
 * gradient. */
NFI_API int nfi_segformer_backward(const nfi_segformer_params *params, const float *g_features,
                                   float *const *grads, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_SEGFORMER_H_ */
