/*
 * nfi_disc_r1.h -- C ABI of the discriminator's R1 regulariser: the double backward of the fused
 * backbone (include/nfi_disc.h) through its image gradient.
 *
 * Reference: run.py's R1 step.  With L = sum_b g_logits[b] logits[b] and the image x,
 *
 *   d_grad_real = dL/dx                 (torch.autograd.grad(..., create_graph=True))
 *   penalty     = mean_b |d_grad_real_b|^2
 *
 * and the penalty's backward hands a cotangent t_img on d_grad_real.  nfi_disc_backward_hvp
 * returns the gradients of Phi = <t_img, J_x^T g_logits>, the directional derivative of L along
 * t_img in image space, with respect to every backbone parameter, the conditioning map cmap, the
 * image (H_xx t_img) and g_logits (J_x t_img, the logits' tangent).  Taken on the saved forward's
 * leaky-ReLU branches (lrelu'' = 0): every layer but the minibatch std is linear there, the
 * first-order cotangents above the minibatch std do not depend on the image (so the 4x4 conv's,
 * fc's and out's bias gradients are exactly zero), and the minibatch std is the one layer with a
 * second-order term.
 *
 * The pass reads the workspace of an nfi_disc_forward with save = 1 and does not write it, so
 * nfi_disc_backward may run before or after it on the same workspace.  Everything else it needs
 * lives in the caller's scratch (nfi_disc_r1_scratch_bytes).  Every sum has a fixed order; there are
 * no atomics.
 *
 * Conventions as in nfi_render.h: device pointers, fp32, stream as void*, 0 = success.
 */
#ifndef NFI_DISC_R1_H_
#define NFI_DISC_R1_H_

#include "nfi_disc.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nfi_disc_hvp {
  const float *g_logits;  /* [B] the first-order cotangent of the logits */
  const float *t_img;     /* [B,nc,R,R] the cotangent of the image gradient */
  void *scratch;          /* at least nfi_disc_r1_scratch_bytes */
  size_t scratch_bytes;
  float *grad_img;        /* [B,nc,R,R] += H_xx t_img, or NULL */
  float *grad_cmap;       /* [B,cmap_dim] +=, or NULL */
  float *grad_g_logits;   /* [B] += J_x t_img, or NULL */
} nfi_disc_hvp;

/* Scratch of nfi_disc_backward_hvp for these sizes (0 on invalid sizes). */
NFI_API size_t nfi_disc_r1_scratch_bytes(const nfi_disc_params *params);
/* After a forward with save = 1 on the same params and workspace: the gradients of
 * <t_img, d(sum g_logits logits)/dimg>, accumulated (+=) into the outputs of `hvp` and into the
 * parameter gradients of `grads` (each optional, NULL: not computed). */
NFI_API int nfi_disc_backward_hvp(const nfi_disc_params *params, const nfi_disc_hvp *hvp,
                                  const nfi_disc_grads *grads, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_DISC_R1_H_ */
