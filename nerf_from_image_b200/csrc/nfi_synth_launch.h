// The narrow entries of the synthesis-network translation unit (nfi_synth.cu), which serve the
// networks other than the synthesis (the LPIPS VGG stack, nfi_lpips.cu; the encoder heads,
// nfi_encoder.cu; the discriminator, nfi_disc.cu; the SegFormer backbone, nfi_segformer.cu).  Every
// kernel they launch is compiled in nfi_synth.cu alone.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>

#include "nfi_pair.cuh"

namespace nfi {
namespace synth {

// Orders of a layer's weight w[co][ci][t] (t: its taps) as a GEMM operand or a weight gradient
enum WeightOrder {
  kTapCoCi,  // [taps][cout][cin]: the conv's B operand
  kTapCiCo,  // [taps][cin][cout]: the data gradient's B operand
  kCoTapCi,  // [cout][taps cin], K index t cin + ci: a conv run as one GEMM over a space-to-depth input
  kCoCiTap,  // [cout][cin][taps]: the weight's own order, as wgrad3x3 and wgrad1x1 leave it
  kCiCoTap,  // [cin][cout][taps]: wgrad_down3x3's transposed gradient
};

// w[co ld + ci taps + t] gain -> the pair `out` in `order` (kTapCoCi, kTapCiCo or kCoTapCi).  With
// gain 1 the pair is split from w's own values.
int prep_weights(const float* w, int cout, int cin, int taps, int ld, float gain, int order, Pair out, cudaStream_t st);

// g_w[co ld + ci taps + t] += gain tmp, tmp in `order` (kCoCiTap, kCiCoTap or kCoTapCi)
int finish_wgrad(const float* tmp, int cout, int cin, int taps, int ld, float gain, int order, float* g_w,
                 cudaStream_t st);

// g_w += gain (the sum over terms k < n of wgrad(k)): each term's weight GEMM adds into tmp (cout cin
// taps floats in `order`, zeroed first), then one finish_wgrad.  The terms are summed before the
// gain, in term order.  A null g_w launches nothing.
template <class Wgrad>
int wgrad_terms(float* g_w, int n, Wgrad&& wgrad, int cout, int cin, int taps, int ld, float gain, int order,
                float* tmp, cudaStream_t st) {
  if (g_w == nullptr) return 0;
  NFI_CUDA(cudaMemsetAsync(tmp, 0, (size_t)cout * cin * taps * sizeof(float), st));
  for (int k = 0; k < n; ++k)
    if (int rc = wgrad(k)) return rc;
  return finish_wgrad(tmp, cout, cin, taps, ld, gain, order, g_w, st);
}

// g_b[c] += sum over chunks k < n_chunks of partial[k C + c], in chunk order.  A null g_b launches
// nothing.
int bias_reduce(const float* partial, int n_chunks, int C, float* g_b, cudaStream_t st);

// src [B][R][Cc] (+ bias[c], where bias is set) -> dst [B][Cc][R], or dst += it with `accumulate`
int transpose(const float* src, int B, int R, int Cc, const float* bias, int accumulate, float* dst, cudaStream_t st);

// A plain stride-1, pad-1 3x3 convolution on conv_tc_kernel.  `in` is [B,H,W,C] as a bf16 pair of
// plain values.
//   conv3x3: weights [9][N][C] (prep_weights, kTapCoCi); u = conv + bias -> u_out (fp32 [B,H,W,N],
//            where set) and, where out.hi is set, relu(u) -> out pair [B,H,W,N]
//   conv3x3_adjoint: the data gradient of such a conv, weights [9][N=Cin][C=Cout] (prep_weights,
//            kTapCiCo), taps flipped -> raw_out fp32 [B,H,W,N]
int conv3x3(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float* u_out, Pair out,
            cudaStream_t st);
int conv3x3_adjoint(int B, int H, int W, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st);

// The weight gradient of such a conv on wgrad_tc_kernel:
//   g_w[co,ci,ky,kx] += sum_{b,y,x} G[b,y,x,co] X[b,y+ky-1,x+kx-1,ci]
// G [B,H,W,g_channels] (the gradient of the conv output; channels >= cout are not read into g_w, so
// a narrow Cout can be zero-padded to the 16-byte TMA row pitch) and X [B,H,W,cin] are bf16 pairs.
// The K split's partial sums go to `partials` (wgrad3x3_partial_floats) and are added to g_w in a
// fixed order: two calls on the same inputs give the same bits.  A null g_w launches nothing.
size_t wgrad3x3_partial_floats(int B, int H, int W, int cout, int cin);
int wgrad3x3(int B, int H, int W, int cout, int cin, int g_channels, Pair g, Pair x, float* partials,
             float* g_w, cudaStream_t st);

// The discriminator's and SegFormer's layers, on the same two kernels:
//   conv3x3_act: conv3x3 with the ACT epilogue's gain and negative slope: lrelu(gain (conv + bias))
//   conv_down3x3: the stride-2 3x3 correlation of a [B,2h+1,2h+1,C] image given as its four parity
//            phases, phase (py,px) at image offset (2py+px) B of a [4B,h+1,h+1,C] pair; weights
//            [9][N][C] (kTapCoCi) -> raw_out fp32 [B,h,h,N]
//   conv_up3x3: its adjoint, the stride-2 transposed conv of [B,h,h,C] with weights [9][N][C]
//            (kTapCiCo of a [C,N,3,3] layer) -> raw_out fp32 [B,2h+1,2h+1,N]
//   conv1x1: [B,H,H,C] against weights [1][N][C] -> raw_out fp32 [B,H,H,N]
//   wgrad_down3x3: conv_down3x3's weight gradient, TRANSPOSED: g_wt[ci,co,ky,kx] += sum over
//            (b,i,j) of phases(ky%2,kx%2)[b, i+ky/2, j+kx/2, ci] g[b,i,j,co]
//   wgrad1x1: g_w[co,ci] += sum over positions of g[.,co] x[.,ci], both [B,H,H,.]
// (the partials and g_w as for wgrad3x3)
int conv3x3_act(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float gain, float slope,
                Pair out, cudaStream_t st);
int conv_down3x3(int B, int h, int C, int N, Pair phases, Pair w, float* raw_out, cudaStream_t st);
int conv_up3x3(int B, int h, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st);
int conv1x1(int B, int H, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st);
size_t wgrad_down3x3_partial_floats(int B, int h, int cin, int cout);
int wgrad_down3x3(int B, int h, int cin, int cout, Pair phases, Pair g, float* partials, float* g_wt, cudaStream_t st);
size_t wgrad1x1_partial_floats(int B, int H, int cout, int cin);
int wgrad1x1(int B, int H, int cout, int cin, Pair g, Pair x, float* partials, float* g_w, cudaStream_t st);
}  // namespace synth
}  // namespace nfi
