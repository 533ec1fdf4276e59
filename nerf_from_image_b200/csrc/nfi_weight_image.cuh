// The plain decoder's weight image (layout: nfi_forward_tc.cuh), in a header of its own so that
// only the units that launch its prep kernel compile it (nfi_render.cu, nfi_pipe.cu).
#pragma once
#include "nfi_forward_tc.cuh"

namespace nfi {

// Builds the weight image: W1 split into TF32 hi/lo and laid out as the wgmma
// B operand ([64 rows = hidden unit][32 k] fp32, K-major, SWIZZLE_128B), W2
// padded to 16 rows with its K positions in register-fragment order (tc::kpos_of_hidden), biases.
static __global__ void prep_weight_image(const float* __restrict__ w1, const float* __restrict__ b1,
                                  const float* __restrict__ w2, const float* __restrict__ b2,
                                  int nout, unsigned char* __restrict__ img, float scale1,
                                  float pad_b2, float scale2) {
  // scale1: factor folded into layer 1 (W1 and b1); pad_b2: value of the padded
  // layer-2 biases; scale2: factor folded into the colour rows (>= 1) of layer 2.  The
  // pipelined kernels want log2(e), -1e30, log2(e) (nfi_forward_pipe.cuh); the stand-alone
  // decoder 1, 0, 1.
  for (int i = threadIdx.x; i < kHid * kC; i += blockDim.x) {
    const int j = i / kC, k = i % kC;  // W1[j][k]
    const float w = w1[i] * scale1;
    const float hi = tc::tf32_hi(w);
    const uint32_t off = tc::sw128_offset(j, k >> 2) + (k & 3) * 4;
    *reinterpret_cast<float*>(img + kWiW1Hi + off) = hi;
    *reinterpret_cast<float*>(img + kWiW1Lo + off) = w - hi;
  }
  for (int i = threadIdx.x; i < kW2Pad * kHid; i += blockDim.x) {
    const int o = i / kHid, j = i % kHid;  // W2[o][j], rows >= nout are zero
    const float w = (o < nout) ? w2[o * kHid + j] * (o >= 1 ? scale2 : 1.f) : 0.f;
    const float hi = tc::tf32_hi(w);
    const int jp = tc::kpos_of_hidden(j);
    const uint32_t off = (jp >> 5) * 2048 + tc::sw128_offset(o, (jp & 31) >> 2) + (jp & 3) * 4;
    *reinterpret_cast<float*>(img + kWiW2Hi + off) = hi;
    *reinterpret_cast<float*>(img + kWiW2Lo + off) = w - hi;
  }
  float* b1i = reinterpret_cast<float*>(img + kWiB1);
  float* b2i = reinterpret_cast<float*>(img + kWiB2);
  for (int i = threadIdx.x; i < kHid; i += blockDim.x) b1i[i] = b1[i] * scale1;
  for (int i = threadIdx.x; i < kW2Pad; i += blockDim.x)
    b2i[i] = (i < nout) ? b2[i] * (i >= 1 ? scale2 : 1.f) : pad_b2;
}

}  // namespace nfi
