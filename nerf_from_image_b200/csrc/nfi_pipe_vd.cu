// Translation unit of the view-direction-conditioned instantiations of the pipelined forward and
// backward kernels (render_forward_pipe / render_backward_pipe<..., VD = true>,
// nfi_forward_pipe.cuh, nfi_backward_pipe.cuh) and their weight images (nfi_layout.h); a unit of
// its own so that build.sh compiles it beside nfi_pipe.cu.
#include "nfi_pipe_ladder.cuh"

namespace nfi {

// The larger weight image and the tile's view features take the forward past the 132 KiB
// carve-out step of the plain kernel (nfi_pipe.cu) to the next one, 164 KiB: 92 KiB of L1 are
// left to the plane gather instead of 124 KiB.
using VdCfg = PipeCfg<3, true>;
static_assert(VdCfg::kSmBytes + kSmemReservedPerCta <= 164 * 1024,
              "render_forward_pipe<VD> no longer fits the 164 KiB carve-out step");
static_assert(VdCfg::kSmA >= kVdBytes && VdCfg::kSmA % 1024 == 0, "weight image overlaps the stages");

// The backward takes the largest carve-out step, 228 KiB: both weight images, three fp32 stages,
// the D2 / dOut and D4 slots, the tile's view features and the rays' view-gradient sums.
using VbCfg = BwdCfg<2, true>;
static_assert(VbCfg::kSmBytes + kSmemReservedPerCta <= kSmemPerSm,
              "render_backward_pipe<VD> no longer fits the 228 KiB carve-out step");
static_assert(VbCfg::kSmWb >= kVdBytes && VbCfg::kSmA - VbCfg::kSmWb >= kVbBytes &&
                  VbCfg::kSmWb % 1024 == 0 && VbCfg::kSmA % 1024 == 0,
              "a weight image overlaps its neighbour in shared memory");

namespace {

__global__ void prep_weight_image_vd(const float* __restrict__ w1, const float* __restrict__ b1,
                                     const float* __restrict__ w2, const float* __restrict__ b2,
                                     const float* __restrict__ w3, const float* __restrict__ b3,
                                     int n_attention, unsigned char* __restrict__ img, float scale1,
                                     float scale3, float pad) {
  vd_weight_image_fill(w1, b1, w2, b2, w3, b3, n_attention, img, scale1, scale3, pad,
                       (int)threadIdx.x, (int)blockDim.x);
}

__global__ void prep_weight_image_vd_bwd(const float* __restrict__ w1, const float* __restrict__ w2,
                                         const float* __restrict__ w3, int n_attention,
                                         unsigned char* __restrict__ img) {
  vd_bwd_weight_image_fill(w1, w2, w3, n_attention, img, (int)threadIdx.x, (int)blockDim.x);
}

}  // namespace

// log2 e goes into layer 1 (the softplus works in log2 units) and, for attention models, into
// W3 / b3: the features pass through a leaky ReLU in natural units, the logits feed a base-2
// softmax whose padded entries sit at -1e30.  The sigmoid colours of A = 0 take natural units.
// The backward image is in natural units throughout (nfi_layout.h).
template <>
int prep_weight_images<true>(const nfi_render_params& p, unsigned char* wimg, bool bwd,
                             cudaStream_t st) {
  const bool att = p.n_attention > 0;
  prep_weight_image_vd<<<1, 256, 0, st>>>(p.w1, p.b1, p.w2, p.b2, p.w3, p.b3, p.n_attention, wimg,
                                          kLog2e, att ? kLog2e : 1.f, att ? kPadLogit : 0.f);
  NFI_CUDA(cudaGetLastError());
  if (bwd) {
    prep_weight_image_vd_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, p.w3, p.n_attention,
                                                wimg + kVdBwdImageOffset);
    NFI_CUDA(cudaGetLastError());
  }
  return 0;
}

template int launch_pipe_forward<true>(const nfi_render_params&, unsigned char*, float*, unsigned,
                                       cudaStream_t);
template int launch_pipe_backward<true>(const nfi_render_params&, const nfi_render_grads&,
                                        unsigned char*, unsigned, cudaStream_t);

}  // namespace nfi
