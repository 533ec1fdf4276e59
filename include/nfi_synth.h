/*
 * nfi_synth.h -- C ABI of the H100 (sm_90a) tri-plane producer: the StyleGAN2 synthesis
 * network that google-research/nerf-from-image runs in front of its per-ray render
 * (SURVEY.md section 8f, N1; the "a5" row of section 8a).
 *
 * Reference: Generator.forward calls `self.synthesis_network(w_synthesis)` and views the result
 * as [B,3,32,R,R] (/root/reference/models/generator.py:475-477).  The network is
 * models/stylegan.py:438-490 (SynthesisNetwork) over SynthesisBlock (:383-435), SynthesisLayer
 * (:293-356: affine -> conv_modulated2d :114-145 -> noise -> bias -> sqrt(2) -> leaky-relu 0.2),
 * OutputLayer (:359-380) and the [1,3,3,1] FIR resamplers (:22-111).  The reference has no FFI;
 * the entry point below is what a ctypes binding of that module call binds
 * (nerf_from_image_b200/synthesis.py), and it emits the planes CHANNEL-LAST ([B,3,R,R,32]), the
 * layout nfi_render_forward gathers from, so no re-layout pass sits between the two.
 *
 * Arithmetic: every convolution is an implicit GEMM on wgmma (bf16 operands: the activations and
 * weights are kept as bf16 hi + lo pairs -- 16 significant bits, 4 bytes per element like the fp32
 * they stand for -- three MMAs per product, fp32 accumulation in registers; the error against the
 * fp64 network is bounded by the tensor core's accumulation, not by the operands; the tests hold it
 * under 3e-4 relative L2 at the full 512-channel size), operands staged by TMA (cp.async.bulk.tensor),
 * prologue (style scaling) folded into the producing layer's epilogue, epilogue (demodulation,
 * noise, bias, gain, leaky-relu, next layer's style, hi/lo split) fused.  Conventions as in nfi_render.h:
 * device pointers, fp32, stream as void*, 0 = success, text via nfi_last_error().
 * Forward only: callers that differentiate through the synthesis network (inversion, GAN
 * training) keep the reference module, which this entry point never falls back to.
 */
#ifndef NFI_SYNTH_H_
#define NFI_SYNTH_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_SYNTH_MAX_BLOCKS 9 /* resolutions 4 .. 1024 */

/* One SynthesisLayer (3x3) or OutputLayer (1x1) -- raw module parameters, no gains folded. */
typedef struct nfi_synth_layer {
  const float *weight;   /* [cout, cin, k, k]                      stylegan.py:317-318,367-368 */
  const float *affine_w; /* [cin, w_dim]  EqualizedLinear.weight   stylegan.py:316,366 */
  const float *affine_b; /* [cin]         EqualizedLinear.bias (init 1) */
  const float *bias;     /* [cout] */
  const float *noise;    /* [B, res, res] ALREADY multiplied by noise_strength (the tensor
                            stylegan.py:334-343 builds), or NULL = no noise for this layer */
} nfi_synth_layer;

typedef struct nfi_synth_params {
  int32_t batch;          /* B */
  int32_t img_resolution; /* R: power of two >= 8 */
  int32_t img_channels;   /* 96 = 3 planes x 32 channels */
  int32_t w_dim;          /* 512 */
  int32_t num_blocks;     /* log2(R) - 1: resolutions 4, 8, ..., R */
  int32_t num_ws;         /* ws.shape[1] >= 2 * num_blocks */
  int32_t channels[NFI_SYNTH_MAX_BLOCKS]; /* feature channels of each block (multiples of 32) */
  const float *ws;          /* [B, num_ws, w_dim] */
  const float *const_input; /* [channels[0], 4, 4]  b4.const */
  nfi_synth_layer conv0[NFI_SYNTH_MAX_BLOCKS]; /* up-sampling layer of block i >= 1 (conv0[0] unused) */
  nfi_synth_layer conv1[NFI_SYNTH_MAX_BLOCKS];
  nfi_synth_layer torgb[NFI_SYNTH_MAX_BLOCKS];
  float *planes;          /* out: [B,3,R,R,32] channel-last tri-planes */
  void *workspace;        /* >= nfi_synthesis_workspace_bytes(params) */
  size_t workspace_bytes;
} nfi_synth_params;

NFI_API size_t nfi_synthesis_workspace_bytes(const nfi_synth_params *params);
NFI_API int nfi_synthesis_forward(const nfi_synth_params *params, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_SYNTH_H_ */
