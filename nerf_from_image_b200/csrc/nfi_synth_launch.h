// Entry points of the synthesis-network translation unit (nfi_synth.cu), compiled in parallel
// with the rest of the library.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_pair.cuh"
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
// (the LPIPS VGG stack, nfi_lpips.cu; the encoder heads, nfi_encoder.cu).  `in` is [B,H,W,C] as a
// bf16 pair of plain values.
//   conv3x3: weights [9][N][C] (prep_weights3x3, transposed 0); u = conv + bias -> u_out (fp32
//            [B,H,W,N], where set) and, where out.hi is set, relu(u) -> out pair [B,H,W,N]
//   conv3x3_adjoint: the data gradient of such a conv, weights [9][N=Cin][C=Cout] (prep_weights3x3,
//            transposed 1), taps flipped -> raw_out fp32 [B,H,W,N]
int conv3x3(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float* u_out, Pair out,
            cudaStream_t st, char* err, size_t err_len);
int conv3x3_adjoint(int B, int H, int W, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st,
                    char* err, size_t err_len);
// weight [Cout,Cin,3,3] -> [9][Cout][Cin] (transposed 0) or [9][Cin][Cout] (transposed 1) pair
int prep_weights3x3(const float* w, int cout, int cin, int transposed, __nv_bfloat16* hi,
                    __nv_bfloat16* lo, cudaStream_t st, char* err, size_t err_len);

// The weight gradient of such a conv on wgrad_tc_kernel (the encoder heads, nfi_encoder.cu):
//   g_w[co,ci,ky,kx] += sum_{b,y,x} G[b,y,x,co] X[b,y+ky-1,x+kx-1,ci]
// G [B,H,W,g_channels] (the gradient of the conv output; channels >= cout are not read into g_w, so
// a narrow Cout can be zero-padded to the 16-byte TMA row pitch) and X [B,H,W,cin] are bf16 pairs.
// The K split's partial sums go to `partials` (wgrad3x3_partial_floats) and are reduced in a fixed
// order: two calls on the same inputs give the same bits.  `w` is the layer's weight (the shared
// reduction reads it; with no demodulation term it does not change the result).  A null g_w
// launches nothing.
size_t wgrad3x3_partial_floats(int B, int H, int W, int cout, int cin);
int wgrad3x3(int B, int H, int W, int cout, int cin, int g_channels, Pair g, Pair x, const float* w,
             float* partials, float* g_w, cudaStream_t st, char* err, size_t err_len);
}  // namespace synth
}  // namespace nfi
