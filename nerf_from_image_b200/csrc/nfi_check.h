// The CUDA-check macro of every launcher in the library, and the warp sum of every unit.  On its own
// so that the render units take them without the bf16-pair header (nfi_pair.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

namespace nfi {
// butterfly: every lane holds the same bits
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
}  // namespace nfi

// A CUDA runtime call in a launcher, which reports into (err, err_len): on failure the call and
// the CUDA error go there and the launcher returns 2.
#define NFI_LAUNCH_CHECK(expr)                                                       \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess) {                                                        \
      snprintf(err, err_len, "%s failed: %s", #expr, cudaGetErrorString(e__));       \
      return 2;                                                                      \
    }                                                                                \
  } while (0)
