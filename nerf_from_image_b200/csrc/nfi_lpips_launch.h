// Entry points of the LPIPS-VGG translation unit (nfi_lpips.cu), compiled in parallel with the rest
// of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_lpips.h"

namespace nfi {
namespace lpips {
size_t workspace_bytes(const nfi_lpips_params& p);
int forward(const nfi_lpips_params& p, cudaStream_t st, char* err, size_t err_len);
int backward(const nfi_lpips_params& p, const float* g_dist, float* grad_in0, float* grad_in1,
             cudaStream_t st, char* err, size_t err_len);
int saved_preactivation(const nfi_lpips_params& p, int layer, float* out, cudaStream_t st, char* err,
                        size_t err_len);
}  // namespace lpips
}  // namespace nfi
