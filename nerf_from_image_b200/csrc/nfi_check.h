// The error channel of every unit in the library, and the warp sum of every unit.  On its own so
// that the render units take them without the bf16-pair header (nfi_pair.cuh).
#pragma once
#include <cuda_runtime.h>

namespace nfi {
// Formats a refusal into the library's thread-local error text (nfi_last_error, defined beside it
// in nfi_render.cu) and returns 1.
int fail(const char* fmt, ...) __attribute__((format(printf, 1, 2)));

// butterfly: every lane holds the same bits
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
}  // namespace nfi

// A CUDA runtime call: on failure the call and the CUDA error go to the error text and the caller
// returns 2.
#define NFI_CUDA(expr)                                                               \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess)                                                          \
      return nfi::fail("%s failed: %s", #expr, cudaGetErrorString(e__)), 2;          \
  } while (0)
