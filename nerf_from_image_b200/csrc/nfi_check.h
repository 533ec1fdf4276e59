// The CUDA-check macro of every launcher in the library.  On its own so that the render units take
// it without the bf16-pair header (nfi_pair.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

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
