// Translation unit of the view-direction-conditioned instantiations of the pipelined forward and
// backward kernels (render_forward_pipe / render_backward_pipe<..., VD = true>,
// nfi_forward_pipe.cuh, nfi_backward_pipe.cuh) and their weight images (nfi_layout.h); a unit of
// its own so that build.sh compiles it beside nfi_pipe.cu.
#include <cuda_runtime.h>
#include <stdio.h>

#include "nfi_backward.cuh"
#include "nfi_backward_pipe.cuh"
#include "nfi_forward_pipe.cuh"
#include "nfi_pipe_launch.h"

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

// The larger weight image and the tile's view features take this kernel past the 132 KiB
// carve-out step of the plain kernel (nfi_pipe.cu) to the next one, 164 KiB: 92 KiB of L1 are
// left to the plane gather instead of 124 KiB.
using VdCfg = PipeCfg<3, true>;
constexpr int kSmemPerSm = 228 * 1024, kSmemReservedPerCta = 1024;
static_assert(VdCfg::kSmBytes + kSmemReservedPerCta <= 164 * 1024,
              "render_forward_pipe<VD> no longer fits the 164 KiB carve-out step");
static_assert(VdCfg::kSmA >= kVdBytes && VdCfg::kSmA % 1024 == 0, "weight image overlaps the stages");
constexpr int kVdCarveoutPct =
    ((VdCfg::kSmBytes + kSmemReservedPerCta) * 100 + kSmemPerSm - 1) / kSmemPerSm;

__global__ void prep_weight_image_vd(const float* __restrict__ w1, const float* __restrict__ b1,
                                     const float* __restrict__ w2, const float* __restrict__ b2,
                                     const float* __restrict__ w3, const float* __restrict__ b3,
                                     int n_attention, unsigned char* __restrict__ img, float scale1,
                                     float scale3, float pad) {
  vd_weight_image_fill(w1, b1, w2, b2, w3, b3, n_attention, img, scale1, scale3, pad,
                       (int)threadIdx.x, (int)blockDim.x);
}

template <int NP, int EX, bool FINE, int NSLOT>
int run_fwd(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
            cudaStream_t st, char* err, size_t err_len) {
  auto k = render_forward_pipe<NP, EX, FINE, 3, false, NSLOT, true>;
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, VdCfg::kSmBytes));
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 kVdCarveoutPct));
  k<<<grid, VdCfg::kThreadsTotal, VdCfg::kSmBytes, st>>>(p, wimg, scratch);
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

template <int NP, int EX>
int fwd_np_ex(const nfi_render_params& p, const unsigned char* wimg, float* scratch, unsigned grid,
              cudaStream_t st, char* err, size_t err_len) {
  if (p.fine_sampling && p.num_samples > 64)  // 4 resampling slots per lane (S <= 128)
    return run_fwd<NP, EX, true, 4>(p, wimg, scratch, grid, st, err, err_len);
  if (p.fine_sampling) return run_fwd<NP, EX, true, 2>(p, wimg, scratch, grid, st, err, err_len);
  return run_fwd<NP, EX, false, 2>(p, wimg, scratch, grid, st, err, err_len);
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

// The backward takes the largest carve-out step, 228 KiB: both weight images, three fp32 stages,
// the D2 / dOut and D4 slots, the tile's view features and the rays' view-gradient sums.
using VbCfg = BwdCfg<2, true>;
static_assert(kVdBackwardWorkspaceBytes == NFI_VIEW_BACKWARD_WORKSPACE_BYTES,
              "nfi_layout.h and nfi_render.h disagree on the view backward's workspace");
static_assert(VbCfg::kSmBytes + kSmemReservedPerCta <= kSmemPerSm,
              "render_backward_pipe<VD> no longer fits the 228 KiB carve-out step");
static_assert(VbCfg::kSmWb >= kVdBytes && VbCfg::kSmA - VbCfg::kSmWb >= kVbBytes &&
                  VbCfg::kSmWb % 1024 == 0 && VbCfg::kSmA % 1024 == 0,
              "a weight image overlaps its neighbour in shared memory");

__global__ void prep_weight_image_vd_bwd(const float* __restrict__ w1, const float* __restrict__ w2,
                                         const float* __restrict__ w3, int n_attention,
                                         unsigned char* __restrict__ img) {
  vd_bwd_weight_image_fill(w1, w2, w3, n_attention, img, (int)threadIdx.x, (int)blockDim.x);
}

template <int NP, int EX, bool CAM>
int run_bwd(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
            unsigned grid, cudaStream_t st, char* err, size_t err_len) {
  auto k = render_backward_pipe<NP, EX, CAM, 2, true>;
  NFI_PCUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, VbCfg::kSmBytes));
  k<<<grid, VbCfg::kThreadsTotal, VbCfg::kSmBytes, st>>>(p, g, wimg);
  NFI_PCUDA(cudaGetLastError());
  return 0;
}

template <int NP>
int bwd_np(const nfi_render_params& p, const nfi_render_grads& g, const unsigned char* wimg,
           unsigned grid, cudaStream_t st, char* err, size_t err_len) {
  const bool cam = g.grad_origins != nullptr;
  if (p.extra_mode == NFI_EXTRA_COORDS && g.g_extra != nullptr)
    return cam ? run_bwd<NP, 1, true>(p, g, wimg, grid, st, err, err_len)
               : run_bwd<NP, 1, false>(p, g, wimg, grid, st, err, err_len);
  return cam ? run_bwd<NP, 0, true>(p, g, wimg, grid, st, err, err_len)
             : run_bwd<NP, 0, false>(p, g, wimg, grid, st, err, err_len);
}

}  // namespace

// log2 e goes into layer 1 (the softplus works in log2 units) and, for attention models, into
// W3 / b3: the features pass through a leaky ReLU in natural units, the logits feed a base-2
// softmax whose padded entries sit at -1e30.  The sigmoid colours of A = 0 take natural units.
int launch_pipe_weight_image_vd(const nfi_render_params& p, unsigned char* wimg, cudaStream_t st) {
  const bool att = p.n_attention > 0;
  prep_weight_image_vd<<<1, 256, 0, st>>>(p.w1, p.b1, p.w2, p.b2, p.w3, p.b3, p.n_attention, wimg,
                                          kLog2e, att ? kLog2e : 1.f, att ? kPadLogit : 0.f);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int launch_pipe_forward_vd(const nfi_render_params& p, int nout_pad, const unsigned char* wimg,
                           float* scratch, unsigned grid, cudaStream_t st, char* err,
                           size_t err_len) {
  if (nout_pad == 4) return fwd_np<4>(p, wimg, scratch, grid, st, err, err_len);
  if (nout_pad == 12) return fwd_np<12>(p, wimg, scratch, grid, st, err, err_len);
  return fwd_np<16>(p, wimg, scratch, grid, st, err, err_len);
}

int launch_pipe_backward_vd(const nfi_render_params& p, const nfi_render_grads& g, int nout_pad,
                            unsigned char* wimg, unsigned grid, cudaStream_t st, char* err,
                            size_t err_len) {
  if (launch_pipe_weight_image_vd(p, wimg, st)) {
    snprintf(err, err_len, "weight image launch failed");
    return 2;
  }
  prep_weight_image_vd_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, p.w3, p.n_attention,
                                              wimg + kVdBwdImageOffset);
  NFI_PCUDA(cudaGetLastError());
  if (nout_pad == 4) return bwd_np<4>(p, g, wimg, grid, st, err, err_len);
  if (nout_pad == 12) return bwd_np<12>(p, g, wimg, grid, st, err, err_len);
  return bwd_np<16>(p, g, wimg, grid, st, err, err_len);
}

}  // namespace nfi
