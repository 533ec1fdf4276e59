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
 * Backward to the latents (the inversion setting: every network parameter frozen):
 * nfi_synthesis_forward_saved runs the same forward -- the same planes, bit for bit -- and also
 * keeps each layer's pre-activation u in the workspace; nfi_synthesis_backward then turns the
 * planes' gradient into the gradient of ws.  Its data-gradient GEMMs run on the same TMA + wgmma
 * kernel with the weights re-laid-out [tap][Cin][Cout]; the up layer's adjoint is the FIR's
 * (a correlation with the same symmetric taps) split into the four parity phases of the
 * (2R+1)^2 raw gradient, then nine stride-1 taps over them.
 * Backward to the parameters (the GAN generator step): nfi_synthesis_backward_params runs the same
 * launches and adds the weight-gradient GEMMs (wgrad_tc_kernel: dL/dconv-output against the
 * layer's input, both position-major bf16 pairs, contracted over positions in bounded tensor-core
 * chains, split over CTAs and reduced in fp32 in a fixed order) and the small reductions for
 * biases, noise, affines and b4.const.  The weight gradients are the same from run to run; the
 * bias sums (one fp32 atomic per block of 1024 positions and image) and the noise sums (shared-
 * memory fp32 atomics over channel groups) are not, in their last bits; g_ws is as reproducible
 * as nfi_synthesis_backward's (the same launches).
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

/* Upstream gradient in, latent gradient out. */
typedef struct nfi_synth_grads {
  const float *g_planes; /* [B,3,R,R,32] channel-last dL/dplanes (nfi_render_backward's grad_planes
                            for channel-last planes) */
  float *g_ws;           /* [B,num_ws,w_dim] ACCUMULATED (+=) like nfi_render_grads */
} nfi_synth_grads;

/* Workspace of a saved forward and the backward that reads it: the forward's buffers, every
   layer's pre-activation (fp32, channel-last) and the backward's scratch. */
NFI_API size_t nfi_synthesis_saved_workspace_bytes(const nfi_synth_params *params);
/* nfi_synthesis_forward, plus the tensors the backward reads, left in params->workspace
   (>= nfi_synthesis_saved_workspace_bytes). */
NFI_API int nfi_synthesis_forward_saved(const nfi_synth_params *params, void *stream);
/* The same params (same ws, weights, noise) and the workspace as the saved forward left it. */
NFI_API int nfi_synthesis_backward(const nfi_synth_params *params, const nfi_synth_grads *grads,
                                   void *stream);
/* Copies one layer's saved pre-activation u (fp32, [B,res,res,cout] channel-last, res = 4 << block)
   out of a saved forward's workspace into `out`: which = 0 is conv0 (block >= 1), 1 is conv1.
   For tests that compare the forward's leaky-ReLU branches with a reference. */
NFI_API int nfi_synthesis_saved_preactivation(const nfi_synth_params *params, int32_t block,
                                              int32_t which, float *out, void *stream);

/* Backward to the parameters (the GAN generator step).  Every pointer is ACCUMULATED (+=) like
   g_ws, has the shape of the nfi_synth_layer field it differentiates, and may be NULL (that
   gradient is not formed). */
typedef struct nfi_synth_layer_grads {
  float *g_weight;   /* [cout, cin, k, k] */
  float *g_affine_w; /* [cin, w_dim] */
  float *g_affine_b; /* [cin] */
  float *g_bias;     /* [cout] */
  float *g_noise;    /* [B, res, res]: gradient of the noise tensor the layer was handed (the value
                        after the multiplication by noise_strength); ignored where noise is NULL */
} nfi_synth_layer_grads;

typedef struct nfi_synth_param_grads {
  nfi_synth_layer_grads conv0[NFI_SYNTH_MAX_BLOCKS]; /* conv0[0] unused */
  nfi_synth_layer_grads conv1[NFI_SYNTH_MAX_BLOCKS];
  nfi_synth_layer_grads torgb[NFI_SYNTH_MAX_BLOCKS]; /* g_noise unused */
  float *g_const;                                    /* [channels[0], 4, 4] b4.const */
} nfi_synth_param_grads;

/* Workspace of a saved forward whose backward also forms the parameter gradients
   (>= nfi_synthesis_saved_workspace_bytes; nfi_synthesis_forward_saved accepts it). */
NFI_API size_t nfi_synthesis_param_workspace_bytes(const nfi_synth_params *params);
/* nfi_synthesis_backward (the same g_ws, bit for bit) plus the parameter gradients; the workspace
   is a saved forward's of >= nfi_synthesis_param_workspace_bytes. */
NFI_API int nfi_synthesis_backward_params(const nfi_synth_params *params,
                                          const nfi_synth_grads *grads,
                                          const nfi_synth_param_grads *param_grads, void *stream);

/* Path-length regulariser (the double backward of generator.py's path_length): with n = g_planes
   the cotangent a first-order nfi_synthesis_backward turned into g_ws = J_ws^T n, and t = t_ws the
   cotangent that arrives on that g_ws, nfi_synthesis_backward_hvp forms the gradient of
   <t, J_ws^T n> with respect to ws (g_ws here, a Hessian-vector product), and, where param_grads
   is not NULL, with respect to every parameter and noise tensor (the same fields as
   nfi_synthesis_backward_params, ACCUMULATED).  It is the tangent of that backward along t: a
   tangent forward pass, then the backward walk beside its tangent on the same GEMM kernels, the
   product and its tangent stacked as 2B images.  params->workspace is a saved forward's and is only
   read, so a later nfi_synthesis_backward_params on it is unaffected. */
typedef struct nfi_synth_hvp {
  const float *g_planes; /* [B,3,R,R,32] the cotangent n that g_ws was formed with */
  const float *t_ws;     /* [B,num_ws,w_dim] cotangent of g_ws; rows the network does not read are ignored */
  float *g_ws;           /* [B,num_ws,w_dim] ACCUMULATED */
  void *scratch;         /* >= nfi_synthesis_hvp_scratch_bytes(params); separate from params->workspace */
  size_t scratch_bytes;
} nfi_synth_hvp;

NFI_API size_t nfi_synthesis_hvp_scratch_bytes(const nfi_synth_params *params);
NFI_API int nfi_synthesis_backward_hvp(const nfi_synth_params *params, const nfi_synth_hvp *hvp,
                                       const nfi_synth_param_grads *param_grads /* may be NULL */,
                                       void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_SYNTH_H_ */
