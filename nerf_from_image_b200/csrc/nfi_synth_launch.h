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

// The discriminator's layers (nfi_disc.cu), on the same two kernels:
//   conv3x3_act: conv3x3 with the ACT epilogue's gain and negative slope: lrelu(gain (conv + bias))
//   conv_down3x3: the stride-2 3x3 correlation of a [B,2h+1,2h+1,C] image given as its four parity
//            phases, phase (py,px) at image offset (2py+px) B of a [4B,h+1,h+1,C] pair; weights
//            [9][N][C] (transposed 0) -> raw_out fp32 [B,h,h,N]
//   conv_up3x3: its adjoint, the stride-2 transposed conv of [B,h,h,C] with weights [9][N][C]
//            (transposed 1 of a [C,N,3,3] layer) -> raw_out fp32 [B,2h+1,2h+1,N]
//   conv1x1: [B,H,H,C] against weights [1][N][C] -> raw_out fp32 [B,H,H,N]
//   wgrad_down3x3: conv_down3x3's weight gradient, TRANSPOSED: g_wt[ci,co,ky,kx] += sum over
//            (b,i,j) of phases(ky%2,kx%2)[b, i+ky/2, j+kx/2, ci] g[b,i,j,co]
//   wgrad1x1: g_w[co,ci] += sum over positions of g[.,co] x[.,ci], both [B,H,H,.]
// (`w` as for wgrad3x3: any buffer of the gradient's size; it does not change the result.)
int conv3x3_act(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float gain, float slope,
                Pair out, cudaStream_t st, char* err, size_t err_len);
int conv_down3x3(int B, int h, int C, int N, Pair phases, Pair w, float* raw_out, cudaStream_t st, char* err,
                 size_t err_len);
int conv_up3x3(int B, int h, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st, char* err,
               size_t err_len);
int conv1x1(int B, int H, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st, char* err,
            size_t err_len);
size_t wgrad_down3x3_partial_floats(int B, int h, int cin, int cout);
int wgrad_down3x3(int B, int h, int cin, int cout, Pair phases, Pair g, const float* w, float* partials,
                  float* g_wt, cudaStream_t st, char* err, size_t err_len);
size_t wgrad1x1_partial_floats(int B, int H, int cout, int cin);
int wgrad1x1(int B, int H, int cout, int cin, Pair g, Pair x, const float* w, float* partials, float* g_w,
             cudaStream_t st, char* err, size_t err_len);
}  // namespace synth
}  // namespace nfi
