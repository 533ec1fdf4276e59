// Translation unit of the pipelined tensor-core kernels: forward (nfi_forward_pipe.cuh),
// backward (nfi_backward_pipe.cuh), surface normals (nfi_normals_pipe.cuh) and decoder-weight
// gradients (nfi_wgrad_pipe.cuh), with the plain decoder's weight images.
#include "nfi_normals_pipe.cuh"
#include "nfi_pipe_ladder.cuh"
#include "nfi_weight_image.cuh"
#include "nfi_wgrad_pipe.cuh"

namespace nfi {

// The plain forward fits the 132 KiB carve-out step, which leaves 124 KiB of L1.  A kernel that
// grows past it takes the 164 KiB step and loses a quarter of that L1.
static_assert(PipeCfg<3>::kSmBytes + kSmemReservedPerCta <= 132 * 1024,
              "render_forward_pipe no longer fits the 132 KiB carve-out step");

// W2^T (padded to K = 32) and W1^T / 3, split into TF32 hi/lo, K-major SWIZZLE_128B.
static __global__ void prep_weight_image_bwd(const float* __restrict__ w1, const float* __restrict__ w2,
                                      int nout, unsigned char* __restrict__ img) {
  for (int i = threadIdx.x; i < kHid * 32; i += blockDim.x) {
    const int j = i / 32, o = i % 32;  // B3[j][o] = W2[o][j]
    const float w = (o < nout) ? w2[o * kHid + j] : 0.f;
    const float hi = tc::tf32_hi(w);
    const uint32_t off = tc::sw128_offset(j, o >> 2) + (o & 3) * 4;
    *reinterpret_cast<float*>(img + kWbW2tHi + off) = hi;
    *reinterpret_cast<float*>(img + kWbW2tLo + off) = w - hi;
  }
  for (int i = threadIdx.x; i < kC * kHid; i += blockDim.x) {
    const int c = i / kHid, j = i % kHid;  // B4[c][j] = W1[j][c] / 3 (features = mean of 3 planes)
    const float w = w1[j * kC + c] * (1.f / 3.f);
    const float hi = tc::tf32_hi(w);
    const int jp = tc::kpos_of_hidden(j);
    const uint32_t off = (jp >> 5) * 4096 + tc::sw128_offset(c, (jp & 31) >> 2) + (jp & 3) * 4;
    *reinterpret_cast<float*>(img + kWbW1tHi + off) = hi;
    *reinterpret_cast<float*>(img + kWbW1tLo + off) = w - hi;
  }
}

// log2 e goes into layer 1 and the colour rows of layer 2; padded logits at -1e30
template <>
int prep_weight_images<false>(const nfi_render_params& p, unsigned char* wimg, bool bwd,
                              cudaStream_t st) {
  const int nout = nout_of(p.n_attention);
  const bool att = p.n_attention > 0;
  prep_weight_image<<<1, 256, 0, st>>>(p.w1, p.b1, p.w2, p.b2, nout, wimg, kLog2e,
                                       att ? kPadLogit : 0.f, att ? kLog2e : 1.f);
  NFI_CUDA(cudaGetLastError());
  if (bwd) {
    prep_weight_image_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, nout, wimg + kBwdImageOffset);
    NFI_CUDA(cudaGetLastError());
  }
  return 0;
}

template int launch_pipe_forward<false>(const nfi_render_params&, unsigned char*, float*, unsigned,
                                        cudaStream_t);
template int launch_pipe_backward<false>(const nfi_render_params&, const nfi_render_grads&,
                                         unsigned char*, unsigned, cudaStream_t);

namespace {

template <int NP, bool PLANES>
int run_wgrad(const nfi_render_params& p, const nfi_render_grads& g, unsigned char* wimg,
              unsigned grid, cudaStream_t st) {
  using Cfg = WgCfgT<PLANES>;
  auto k = render_wgrad_pipe<NP, PLANES>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmBytes));
  k<<<grid, Cfg::kThreadsTotal, Cfg::kSmBytes, st>>>(p, g, wimg,
                                                     reinterpret_cast<float*>(wimg + kWgAccOffset));
  NFI_CUDA(cudaGetLastError());
  return 0;
}

template <bool PLANES>
int wgrad_np(const nfi_render_params& p, const nfi_render_grads& g, unsigned char* wimg,
             unsigned grid, cudaStream_t st) {
  switch (nout_pad_of(p.n_attention)) {
    case 4: return run_wgrad<4, PLANES>(p, g, wimg, grid, st);
    case 12: return run_wgrad<12, PLANES>(p, g, wimg, grid, st);
    default: return run_wgrad<16, PLANES>(p, g, wimg, grid, st);
  }
}

}  // namespace

size_t pipe_scratch_bytes_per_cta(int num_samples, int nes) {
  return pipe_scratch_floats(num_samples, nes) * sizeof(float);
}

int launch_pipe_wgrad(const nfi_render_params& p, const nfi_render_grads& g, unsigned char* wimg,
                      unsigned grid, bool planes, cudaStream_t st) {
  if (int rc = prep_weight_images<false>(p, wimg, true, st)) return rc;
  return planes ? wgrad_np<true>(p, g, wimg, grid, st) : wgrad_np<false>(p, g, wimg, grid, st);
}

int launch_pipe_normals(const nfi_render_params& p, unsigned char* wimg, unsigned char* wimg_bwd,
                        unsigned grid, cudaStream_t st) {
  // render_normals_pipe needs layer 1 and the distance row of the plain image: row 0 of w2 with
  // or without a view.  A view render is done with its own image (stream order), so the plain
  // one takes its place.
  if (p.view_features)
    if (int rc = prep_weight_images<false>(p, wimg, false, st)) return rc;
  prep_weight_image_bwd<<<1, 256, 0, st>>>(p.w1, p.w2, nout_of(p.n_attention), wimg_bwd);
  NFI_CUDA(cudaGetLastError());
  NFI_CUDA(cudaMemsetAsync(p.normals, 0,
                           (size_t)p.batch * p.height * p.width * 3 * sizeof(float), st));
  using Cfg = BwdCfg<2>;
  constexpr int smem = Cfg::kSmBytes + (kBwdSlots * 128 + kHid) * (int)sizeof(float);
#define NFI_NRM(NP)                                                                          \
  do {                                                                                       \
    auto k = render_normals_pipe<NP, 2>;                                                     \
    NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));    \
    k<<<grid, Cfg::kThreadsTotal, smem, st>>>(p, wimg, wimg_bwd);                            \
  } while (0)
  const int np = nout_pad_of(p.n_attention);
  if (np == 4) NFI_NRM(4); else if (np == 12) NFI_NRM(12); else NFI_NRM(16);
#undef NFI_NRM
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace nfi
