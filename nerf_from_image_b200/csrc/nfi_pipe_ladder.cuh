// Launch ladders of the pipelined forward and backward kernels, templated on VD (view
// conditioning): nfi_pipe.cu instantiates them for the plain decoder and nfi_pipe_vd.cu for the
// view-conditioned one, each beside the prep kernels of its weight images.
#pragma once
#include <cuda_runtime.h>

#include "nfi_backward_pipe.cuh"
#include "nfi_pipe_launch.h"
#include "nfi_route.h"

namespace nfi {

// The forward's plane gather runs out of L1, and on Hopper L1 gets what the shared-memory carve-out
// leaves of 256 KiB.  The carve-out comes in steps (..., 100, 132, 164, 196, 228 KiB), and the
// driver reserves 1 KiB per CTA.
constexpr int kSmemPerSm = 228 * 1024, kSmemReservedPerCta = 1024;
// the smallest carve-out (percent of kSmemPerSm) that holds `smem` bytes: the driver rounds it up
// to the next step
constexpr int carveout_pct(int smem) {
  return ((smem + kSmemReservedPerCta) * 100 + kSmemPerSm - 1) / kSmemPerSm;
}

// The forward weight image at `wimg` and, with `bwd`, the backward image behind it; defined beside
// the prep kernels (nfi_pipe.cu, nfi_pipe_vd.cu).
template <bool VD>
int prep_weight_images(const nfi_render_params& p, unsigned char* wimg, bool bwd, cudaStream_t st);

namespace ladder {

template <int NP, int EX, bool FINE, bool DBG, int NSLOT, bool VD>
int run_fwd(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
            cudaStream_t st) {
  using Cfg = PipeCfg<3, VD>;
  auto k = render_forward_pipe<NP, EX, FINE, 3, DBG, NSLOT, VD>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmBytes));
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout,
                                carveout_pct(Cfg::kSmBytes)));
  k<<<grid, Cfg::kThreadsTotal, Cfg::kSmBytes, st>>>(p, wimg, scratch);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

template <int NP, int EX, bool VD>
int fwd_np_ex(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
              cudaStream_t st) {
  if constexpr (!VD && NP == 12 && EX == 0) {
    if ((p.mlp_mode & kDbgPhaseTimers) && p.fine_sampling)  // tools/phase_times_pipe.py
      return run_fwd<NP, EX, true, true, 2, VD>(p, wimg, scratch, grid, st);
  }
  if (p.fine_sampling && p.num_samples > 64)  // 4 resampling slots per lane (S <= 128)
    return run_fwd<NP, EX, true, false, 4, VD>(p, wimg, scratch, grid, st);
  if (p.fine_sampling)
    return run_fwd<NP, EX, true, false, 2, VD>(p, wimg, scratch, grid, st);
  return run_fwd<NP, EX, false, false, 2, VD>(p, wimg, scratch, grid, st);
}

template <int NP, bool VD>
int fwd_np(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
           cudaStream_t st) {
  if (p.extra_mode == NFI_EXTRA_COORDS)
    return fwd_np_ex<NP, 1, VD>(p, wimg, scratch, grid, st);
  if constexpr (NP > 4) {
    if (p.extra_mode == NFI_EXTRA_SEMANTICS)
      return fwd_np_ex<NP, 2, VD>(p, wimg, scratch, grid, st);
  }
  return fwd_np_ex<NP, 0, VD>(p, wimg, scratch, grid, st);
}

template <int NP, int EX, bool CAM, bool VD>
int run_bwd(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
            unsigned grid, cudaStream_t st) {
  using Cfg = BwdCfg<2, VD>;
  auto k = render_backward_pipe<NP, EX, CAM, 2, VD>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmBytes));
  k<<<grid, Cfg::kThreadsTotal, Cfg::kSmBytes, st>>>(p, g, wimg);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

template <int NP, bool VD>
int bwd_np(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
           unsigned grid, cudaStream_t st) {
  const bool cam = g.grad_origins != nullptr;
  if (p.extra_mode == NFI_EXTRA_COORDS && g.g_extra != nullptr)
    return cam ? run_bwd<NP, 1, true, VD>(p, g, wimg, grid, st)
               : run_bwd<NP, 1, false, VD>(p, g, wimg, grid, st);
  return cam ? run_bwd<NP, 0, true, VD>(p, g, wimg, grid, st)
             : run_bwd<NP, 0, false, VD>(p, g, wimg, grid, st);
}

}  // namespace ladder

template <bool VD>
int launch_pipe_forward(const nfi_render_params& p, unsigned char* wimg, float* scratch,
                        unsigned grid, cudaStream_t st) {
  if (int rc = prep_weight_images<VD>(p, wimg, false, st)) return rc;
  switch (nout_pad_of(p.n_attention)) {
    case 4: return ladder::fwd_np<4, VD>(p, wimg, scratch, grid, st);
    case 12: return ladder::fwd_np<12, VD>(p, wimg, scratch, grid, st);
    default: return ladder::fwd_np<16, VD>(p, wimg, scratch, grid, st);
  }
}

template <bool VD>
int launch_pipe_backward(const nfi_render_params& p, const nfi_render_grads& g,
                         unsigned char* wimg, unsigned grid, cudaStream_t st) {
  if (int rc = prep_weight_images<VD>(p, wimg, true, st)) return rc;
  switch (nout_pad_of(p.n_attention)) {
    case 4: return ladder::bwd_np<4, VD>(p, g, wimg, grid, st);
    case 12: return ladder::bwd_np<12, VD>(p, g, wimg, grid, st);
    default: return ladder::bwd_np<16, VD>(p, g, wimg, grid, st);
  }
}

}  // namespace nfi
