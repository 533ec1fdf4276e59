// What the units on the synthesis network's bf16-pair conv kernels share (nfi_synth.cu, nfi_lpips.cu,
// nfi_encoder.cu, nfi_disc.cu, nfi_segformer.cu): the pair split, the small device helpers, the
// workspace walk and the launch-grid helpers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nfi_check.h"

namespace nfi {

// t = hi + lo with hi = bf16(t), lo = bf16(t - hi)
__device__ __forceinline__ void split_bf16(float t, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(t);
  lo = __float2bfloat16_rn(t - __bfloat162float(hi));
}
__device__ __forceinline__ float relu(float x) { return x > 0.f ? x : 0.f; }
__device__ __forceinline__ float lrelu(float x, float slope) { return x > 0.f ? x : slope * x; }
// lrelu' at the pre-activation u
__device__ __forceinline__ float lrelu_grad(float u, float slope) { return u > 0.f ? 1.f : slope; }

// PyTorch's upsample_bilinear2d source index for align_corners=False with a given scale factor
// (area_pixel_compute_source_index with scale 1 / factor): the two taps and their weights
__device__ __forceinline__ void src_index(int dst, float inv_s, int in, int& i0, int& i1, float& l0, float& l1) {
  float s = inv_s * ((float)dst + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = s - (float)i0;
  l0 = 1.f - l1;
}
// The weight with which destination index `dst` reads source index `src` (both taps may be `src`
// at the clamped last row)
__device__ __forceinline__ float src_weight(int dst, int src, float inv_s, int in) {
  int i0, i1;
  float l0, l1;
  src_index(dst, inv_s, in, i0, i1, l0, l1);
  return (i0 == src ? l0 : 0.f) + (i1 == src ? l1 : 0.f);
}

// A tensor as two bf16 tensors of its shape, hi and lo of split_bf16
struct Pair {
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
};

// The workspace as a deterministic walk: each take is rounded up to 1024 bytes, so every tensor
// starts on a 1024-byte boundary of an aligned base.  With a null base it only counts (the sizers).
struct Bump {
  unsigned char* base;
  size_t off, cap;
  float* take(size_t floats) {
    const size_t bytes = (floats * sizeof(float) + 1023) & ~(size_t)1023;
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += bytes;
    return p;
  }
  Pair pair(size_t elems) {  // two bf16 tensors of `elems` elements
    Pair p;
    p.hi = reinterpret_cast<__nv_bfloat16*>(take((elems + 1) / 2));
    p.lo = reinterpret_cast<__nv_bfloat16*>(take((elems + 1) / 2));
    return p;
  }
};

// A Bump over a caller's buffer from its first 1024-byte boundary (the sizers add the 1024 bytes)
inline Bump aligned_bump(void* p, size_t bytes) {
  unsigned char* base =
      reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
  return Bump{base, 0, bytes};
}

inline int sm_count() {
  static int n = []() {
    int dev = 0, v = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();
  return n;
}

inline unsigned blocks(size_t n, int per) { return (unsigned)((n + per - 1) / per); }
// The grid of a grid-stride kernel over n items: one thread each, at most 16 blocks of 256 per SM
inline unsigned flat_grid(size_t n) {
  const unsigned g = blocks(n, 256), cap = (unsigned)sm_count() * 16u;
  return g > cap ? cap : g;
}

}  // namespace nfi
