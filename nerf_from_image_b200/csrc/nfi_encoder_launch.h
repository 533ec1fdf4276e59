// Entry points of the encoder-heads translation unit (nfi_encoder.cu), compiled in parallel with the
// rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_encoder.h"

namespace nfi {
namespace encoder {
size_t workspace_bytes(const nfi_encoder_params& p);
int forward(const nfi_encoder_params& p, cudaStream_t st, char* err, size_t err_len);
int backward(const nfi_encoder_params& p, const float* g_maps, const float* g_pooled,
             const nfi_encoder_grads& g, cudaStream_t st, char* err, size_t err_len);
int saved_activation(const nfi_encoder_params& p, int layer, float* out, cudaStream_t st, char* err,
                     size_t err_len);
}  // namespace encoder
}  // namespace nfi
