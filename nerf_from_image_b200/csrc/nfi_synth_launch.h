// Entry points of the synthesis-network translation unit (nfi_synth.cu), compiled in parallel
// with the rest of the library.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_synth.h"

namespace nfi {
namespace synth {
size_t workspace_bytes(const nfi_synth_params& p);
int forward(const nfi_synth_params& p, cudaStream_t st, char* err, size_t err_len);
size_t saved_workspace_bytes(const nfi_synth_params& p);
int forward_saved(const nfi_synth_params& p, cudaStream_t st, char* err, size_t err_len);
int backward(const nfi_synth_params& p, const nfi_synth_grads& g, cudaStream_t st, char* err,
             size_t err_len);
size_t param_workspace_bytes(const nfi_synth_params& p);
int backward_params(const nfi_synth_params& p, const nfi_synth_grads& g,
                    const nfi_synth_param_grads& pg, cudaStream_t st, char* err, size_t err_len);
}  // namespace synth
}  // namespace nfi
