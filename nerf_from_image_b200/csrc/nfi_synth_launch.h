// Entry points of the synthesis-network translation unit (nfi_synth.cu), compiled in parallel
// with the rest of the library.
#pragma once
#include <cuda_bf16.h>
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
int saved_preactivation(const nfi_synth_params& p, int block, int which, float* out, cudaStream_t st,
                        char* err, size_t err_len);
size_t param_workspace_bytes(const nfi_synth_params& p);
int backward_params(const nfi_synth_params& p, const nfi_synth_grads& g,
                    const nfi_synth_param_grads& pg, cudaStream_t st, char* err, size_t err_len);
size_t hvp_scratch_bytes(const nfi_synth_params& p);
int backward_hvp(const nfi_synth_params& p, const nfi_synth_hvp& h, const nfi_synth_param_grads* pg,
                 cudaStream_t st, char* err, size_t err_len);

// A plain stride-1, pad-1 3x3 convolution on conv_tc_kernel, for networks other than the synthesis
// (the LPIPS VGG stack, nfi_lpips.cu).  `in` is [B,H,W,C] as a bf16 pair of plain values.
//   forward (adjoint 0): weights [9][N][C] (prep_weights, transposed 0); u = conv + bias -> u_out
//            (fp32 [B,H,W,N]) and, where out_hi is set, relu(u) -> out pair [B,H,W,N]
//   adjoint (adjoint 1): the data gradient of such a conv, weights [9][N=Cin][C=Cout] (prep_weights,
//            transposed 1), taps flipped -> raw_out fp32 [B,H,W,N]
struct Conv3x3 {
  int B, H, W, C, N;
  const __nv_bfloat16* in_hi;
  const __nv_bfloat16* in_lo;
  const __nv_bfloat16* w_hi;
  const __nv_bfloat16* w_lo;
  int adjoint;
  const float* bias;
  float* u_out;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  float* raw_out;
};
int conv3x3(const Conv3x3& c, cudaStream_t st, char* err, size_t err_len);
// weight [Cout,Cin,3,3] -> [9][Cout][Cin] (transposed 0) or [9][Cin][Cout] (transposed 1) pair
int prep_weights3x3(const float* w, int cout, int cin, int transposed, __nv_bfloat16* hi,
                    __nv_bfloat16* lo, cudaStream_t st, char* err, size_t err_len);
}  // namespace synth
}  // namespace nfi
