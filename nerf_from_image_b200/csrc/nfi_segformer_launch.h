// Entry points of the SegFormer-backbone translation unit (nfi_segformer.cu), compiled in parallel
// with the rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_segformer.h"

namespace nfi {
namespace segformer {
size_t workspace_bytes(const nfi_segformer_params& p);
int forward(const nfi_segformer_params& p, cudaStream_t st, char* err, size_t err_len);
int backward(const nfi_segformer_params& p, const float* g_features, float* const* grads, cudaStream_t st,
             char* err, size_t err_len);
}  // namespace segformer
}  // namespace nfi
