// Entry points of the discriminator translation unit (nfi_disc.cu), compiled in parallel with the
// rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_disc.h"
#include "nfi_disc_r1.h"

namespace nfi {
namespace disc {
size_t workspace_bytes(const nfi_disc_params& p);
int forward(const nfi_disc_params& p, cudaStream_t st, char* err, size_t err_len);
int backward(const nfi_disc_params& p, const float* g_logits, float* grad_img, float* grad_cmap,
             const nfi_disc_grads& g, cudaStream_t st, char* err, size_t err_len);
int saved_preactivation(const nfi_disc_params& p, int block, int which, float* out, cudaStream_t st, char* err,
                        size_t err_len);
size_t hvp_scratch_bytes(const nfi_disc_params& p);
int backward_hvp(const nfi_disc_params& p, const nfi_disc_hvp& h, const nfi_disc_grads& g, cudaStream_t st,
                 char* err, size_t err_len);
}  // namespace disc
}  // namespace nfi
