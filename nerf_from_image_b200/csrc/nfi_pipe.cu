// Translation unit of the pipelined tensor-core kernels: forward (nfi_forward_pipe.cuh),
// backward (nfi_backward_pipe.cuh), surface normals (nfi_normals_pipe.cuh) and decoder-weight
// gradients (nfi_wgrad_pipe.cuh).
#include <cuda_runtime.h>
#include <stdio.h>

#include "nfi_backward.cuh"
#include "nfi_backward_pipe.cuh"
#include "nfi_forward_pipe.cuh"
#include "nfi_normals_pipe.cuh"
#include "nfi_pipe_launch.h"
#include "nfi_wgrad_pipe.cuh"

namespace nfi {
namespace {

#define NFI_PCUDA(expr)                                                              \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess) {                                                        \
      snprintf(err, err_len, "%s failed: %s", #expr, cudaGetErrorString(e__));       \
      return 2;                                                                      \
    }                                                                                \
  } while (0)

// The forward's plane gather runs out of L1, and on Hopper L1 gets what the shared-memory carve-out
// leaves of 256 KiB.  The carve-out comes in steps (..., 100, 132, 164, 196, 228 KiB); with the
// 1 KiB the driver reserves per CTA the forward fits the 132 KiB step, which leaves 124 KiB of L1.
// A kernel that grows past it takes the 164 KiB step and loses a quarter of that L1.
constexpr int kSmemPerSm = 228 * 1024, kSmemReservedPerCta = 1024;
static_assert(PipeCfg<3>::kSmBytes + kSmemReservedPerCta <= 132 * 1024,
              "render_forward_pipe no longer fits the 132 KiB carve-out step");
// the smallest carve-out (percent of kSmemPerSm) that holds the kernel: the driver rounds it up
// to the next step
constexpr int kFwdCarveoutPct =
    ((PipeCfg<3>::kSmBytes + kSmemReservedPerCta) * 100 + kSmemPerSm - 1) / kSmemPerSm;

template <int NP, int EX, bool FINE, bool DBG, int NSLOT>
int run_fwd(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
            cudaStream_t st, char* err, size_t err_len) {
  auto k = render_forward_pipe<NP, EX, FINE, 3, DBG, NSLOT>;
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 PipeCfg<3>::kSmBytes));
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 kFwdCarveoutPct));
  k<<<grid, PipeCfg<3>::kThreadsTotal, PipeCfg<3>::kSmBytes, st>>>(p, wimg, scratch);
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

template <int NP, int EX>
int fwd_np_ex(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
              cudaStream_t st, char* err, size_t err_len) {
  if constexpr (NP == 12 && EX == 0) {
    if ((p.mlp_mode & 0x1000) && p.fine_sampling)  // phase-timer build (tools/phase_times_pipe.py)
      return run_fwd<NP, EX, true, true, 2>(p, wimg, scratch, grid, st, err, err_len);
  }
  if (p.fine_sampling && p.num_samples > 64)  // 4 resampling slots per lane (S <= 128)
    return run_fwd<NP, EX, true, false, 4>(p, wimg, scratch, grid, st, err, err_len);
  if (p.fine_sampling) return run_fwd<NP, EX, true, false, 2>(p, wimg, scratch, grid, st, err, err_len);
  return run_fwd<NP, EX, false, false, 2>(p, wimg, scratch, grid, st, err, err_len);
}

template <int NP>
int fwd_np(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
           cudaStream_t st, char* err, size_t err_len) {
  if (p.extra_mode == NFI_EXTRA_COORDS)
    return fwd_np_ex<NP, 1>(p, wimg, scratch, grid, st, err, err_len);
  if constexpr (NP > 4) {
    if (p.extra_mode == NFI_EXTRA_SEMANTICS)
      return fwd_np_ex<NP, 2>(p, wimg, scratch, grid, st, err, err_len);
  }
  return fwd_np_ex<NP, 0>(p, wimg, scratch, grid, st, err, err_len);
}

template <int NP, int EX, bool CAM>
int run_bwd(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
            unsigned grid, cudaStream_t st, char* err, size_t err_len) {
  using Cfg = BwdCfg<2>;
  auto k = render_backward_pipe<NP, EX, CAM, 2>;
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmBytes));
  k<<<grid, Cfg::kThreadsTotal, Cfg::kSmBytes, st>>>(p, g, wimg);
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

template <int NP>
int bwd_np(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
           unsigned grid, cudaStream_t st, char* err, size_t err_len) {
  const bool cam = g.grad_origins != nullptr;
  const bool coords = p.extra_mode == NFI_EXTRA_COORDS && g.g_extra != nullptr;
  if (coords)
    return cam ? run_bwd<NP, 1, true>(p, g, wimg, grid, st, err, err_len)
               : run_bwd<NP, 1, false>(p, g, wimg, grid, st, err, err_len);
  return cam ? run_bwd<NP, 0, true>(p, g, wimg, grid, st, err, err_len)
             : run_bwd<NP, 0, false>(p, g, wimg, grid, st, err, err_len);
}

template <int NP, bool PLANES>
int run_wgrad(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
              unsigned grid, cudaStream_t st, char* err, size_t err_len) {
  using Cfg = WgCfgT<PLANES>;
  auto k = render_wgrad_pipe<NP, PLANES>;
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmBytes));
  k<<<grid, Cfg::kThreadsTotal, Cfg::kSmBytes, st>>>(
      p, g, wimg, reinterpret_cast<float*>(const_cast<unsigned char*>(wimg) + 65536));
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

}  // namespace

size_t pipe_wgrad_workspace_bytes(unsigned grid) { return 65536 + (size_t)grid * kWgAccBytesPerCta; }

size_t pipe_scratch_bytes_per_cta(int num_samples, int nes) {
  return pipe_scratch_floats(num_samples, nes) * sizeof(float);
}

int launch_pipe_weight_image(const nfi_render_params& p, unsigned char* wimg, cudaStream_t st) {
  const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  prep_weight_image<<<1, 256, 0, st>>>(p.w1, p.b1, p.w2, p.b2, nout, wimg, kLog2e,
                                       p.n_attention > 0 ? kPadLogit : 0.f,
                                       p.n_attention > 0 ? kLog2e : 1.f);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int launch_pipe_forward(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                        float* scratch, unsigned grid, cudaStream_t st, char* err,
                        size_t err_len) {
  if (nout_pad == 4) return fwd_np<4>(p, wimg, scratch, grid, st, err, err_len);
  if (nout_pad == 12) return fwd_np<12>(p, wimg, scratch, grid, st, err, err_len);
  return fwd_np<16>(p, wimg, scratch, grid, st, err, err_len);
}

int launch_pipe_backward(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                         unsigned char* wimg, unsigned grid, cudaStream_t st, char* err,
                         size_t err_len) {
  const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  if (launch_pipe_weight_image(p, wimg, st)) {
    snprintf(err, err_len, "weight image launch failed");
    return 2;
  }
  prep_weight_image_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, nout, wimg + 32768);
  NFI_PCUDA(cudaGetLastError());
  if (nout_pad == 4) return bwd_np<4>(p, g, wimg, grid, st, err, err_len);
  if (nout_pad == 12) return bwd_np<12>(p, g, wimg, grid, st, err, err_len);
  return bwd_np<16>(p, g, wimg, grid, st, err, err_len);
}

// decoder-weight gradients on the tensor cores (nfi_wgrad_pipe.cuh): both weight images +
// render_wgrad_pipe
int launch_pipe_wgrad(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                      unsigned char* wimg, unsigned grid, bool planes, cudaStream_t st, char* err,
                      size_t err_len) {
  const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  if (launch_pipe_weight_image(p, wimg, st)) {
    snprintf(err, err_len, "weight image launch failed");
    return 2;
  }
  prep_weight_image_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, nout, wimg + 32768);
  NFI_PCUDA(cudaGetLastError());
  if (planes) {
    if (nout_pad == 4) return run_wgrad<4, true>(p, g, wimg, grid, st, err, err_len);
    if (nout_pad == 12) return run_wgrad<12, true>(p, g, wimg, grid, st, err, err_len);
    return run_wgrad<16, true>(p, g, wimg, grid, st, err, err_len);
  }
  if (nout_pad == 4) return run_wgrad<4, false>(p, g, wimg, grid, st, err, err_len);
  if (nout_pad == 12) return run_wgrad<12, false>(p, g, wimg, grid, st, err, err_len);
  return run_wgrad<16, false>(p, g, wimg, grid, st, err, err_len);
}

// surface normals after render_forward_pipe (nfi_normals_pipe.cuh): `wimg` = the forward weight
// image of that launch, `wimg_bwd` = 32 KiB for the backward image (W1^T / 3 is what is used)
int launch_pipe_normals(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                        unsigned char* wimg_bwd, unsigned grid, cudaStream_t st, char* err,
                        size_t err_len) {
  const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  prep_weight_image_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, nout, wimg_bwd);
  NFI_PCUDA(cudaGetLastError());
  NFI_PCUDA(cudaMemsetAsync(p.normals, 0,
                            (size_t)p.batch * p.height * p.width * 3 * sizeof(float), st));
  using Cfg = BwdCfg<2>;
  constexpr int smem = Cfg::kSmBytes + (kBwdSlots * 128 + kHid) * (int)sizeof(float);
#define NFI_NRM(NP)                                                                          \
  do {                                                                                       \
    auto k = render_normals_pipe<NP, 2>;                                                     \
    NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));   \
    k<<<grid, Cfg::kThreadsTotal, smem, st>>>(p, wimg, wimg_bwd);                            \
  } while (0)
  if (nout_pad == 4) NFI_NRM(4); else if (nout_pad == 12) NFI_NRM(12); else NFI_NRM(16);
#undef NFI_NRM
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

}  // namespace nfi
