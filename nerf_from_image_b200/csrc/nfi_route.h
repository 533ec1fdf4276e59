// Which kernels a render request runs on: the routing policy of nfi_render_forward /
// nfi_render_backward (nfi_render.cu), and the workspace sizes it compares against.  Host-only and
// compilable by a host C++ compiler without the CUDA toolkit (tests/c/route_check.cpp pins a table
// of requests to their routes).
#pragma once
#include "nfi_layout.h"
#include "nfi_render.h"

namespace nfi {

// mlp_mode: the enum nfi_mlp_mode in the low byte, and debug bits
constexpr int kMlpModeMask = 0xff;
// p.normals is the phase-timer buffer of render_forward_pipe's DBG instantiation
// (tools/phase_times_pipe.py), not a normals output
constexpr int kDbgPhaseTimers = 0x1000;
// decoder gradients in two sweeps even without a pose gradient (tools/time_wgrad.py)
constexpr int kDbgTwoSweeps = 0x2000;

static_assert(kWgAccOffset + kMaxPersistentCtas * kWgAccBytesPerCta ==
                  (size_t)NFI_BACKWARD_WORKSPACE_BYTES,
              "nfi_layout.h and nfi_render.h disagree on the backward's workspace");
static_assert(kVdBackwardWorkspaceBytes == NFI_VIEW_BACKWARD_WORKSPACE_BYTES,
              "nfi_layout.h and nfi_render.h disagree on the view backward's workspace");

enum class Route {
  kPipe,             // render_forward_pipe / render_backward_pipe
  kPipeVd,           // their view-conditioned instantiations
  kSimt,             // render_forward_simt / render_backward_simt
  kSimtVd,           // their view-conditioned instantiations
  kWgradOneSweep,    // render_wgrad_pipe<PLANES>: the whole backward in one sweep
  kPipeAndWgrad,     // render_backward_pipe, then render_wgrad_pipe<false>
  kWgrad,            // render_wgrad_pipe<false> alone
  kRefused,
};

struct Plan {
  Route route;
  bool normals_pipe;    // forward: render_normals_pipe runs after the render
  const char* refusal;  // kRefused: the error text
};

inline bool wants_normals(const nfi_render_params& p) {
  return p.compute_normals && !(p.mlp_mode & kDbgPhaseTimers);
}

// The envelope of the pipelined kernels: <= 4 samples per lane in the resampler and float4
// jitter; semantics only with NOUT_PAD > 4 (palettes of <= 3 entries stay on the SIMT kernel)
inline bool in_pipe_envelope(const nfi_render_params& p) {
  return p.num_samples <= 128 && p.num_samples % 4 == 0 &&
         !(p.extra_mode == NFI_EXTRA_SEMANTICS && p.n_attention <= 3);
}

// Forward: the modes that take the pipelined kernels (NFI_MLP_TC_3XTF32 and NFI_MLP_TC_WARPSPEC
// are aliases of NFI_MLP_TC_PIPE) inside the envelope.  Surface normals run on a second pipelined
// kernel (nfi_normals_pipe.cuh), which walks the merged samples and so needs the fine depths, and
// does not write to peers; else the SIMT kernel takes them.
inline Plan route_forward(const nfi_render_params& p) {
  const int mode = p.mlp_mode & kMlpModeMask;
  const bool tc_mode = mode == NFI_MLP_AUTO || mode == NFI_MLP_TC_3XTF32 ||
                       mode == NFI_MLP_TC_WARPSPEC || mode == NFI_MLP_TC_PIPE;
  const bool normals = wants_normals(p);
  const bool pipe = tc_mode && in_pipe_envelope(p) &&
                    (!normals || ((!p.fine_sampling || p.z_fine != nullptr) && p.n_peers == 0));
  if (pipe) return {p.view_features ? Route::kPipeVd : Route::kPipe, normals, nullptr};
  if (tc_mode && mode != NFI_MLP_AUTO)
    return {Route::kRefused, false,
            "tensor-core modes need S <= 128 and S % 4 == 0 and no semantics output; "
            "use NFI_MLP_AUTO"};
  if (p.n_peers > 0)
    return {Route::kRefused, false, "peer outputs (n_peers > 0) need the pipelined kernel"};
  return {p.view_features ? Route::kSimtVd : Route::kSimt, false, nullptr};
}

// Backward, for requests that passed nfi_render_backward's argument checks.  The pipelined
// kernels want any mode but NFI_MLP_FP32_SIMT, the envelope, no semantics output at all and a
// workspace for their weight images; outside that the SIMT kernel runs (no refusal).  Decoder
// gradients (the GAN generator step) run on render_wgrad_pipe, which needs the accumulator rows
// of NFI_BACKWARD_WORKSPACE_BYTES and no upstream gradient of the coords output.  A view-
// conditioned render takes render_backward_pipe<VD> only with decoder and mapper frozen.
inline Plan route_backward(const nfi_render_params& p, const nfi_render_grads& g) {
  const bool env = (p.mlp_mode & kMlpModeMask) != NFI_MLP_FP32_SIMT && in_pipe_envelope(p) &&
                   p.extra_mode != NFI_EXTRA_SEMANTICS && p.workspace != nullptr;
  const bool wgrad = g.grad_w1 || g.grad_b1 || g.grad_w2 || g.grad_b2;
  if (p.view_features) {
    const bool pipe = env && !wgrad && !g.grad_w3 && !g.grad_b3 &&
                      p.workspace_bytes >= (size_t)NFI_VIEW_BACKWARD_WORKSPACE_BYTES;
    return {pipe ? Route::kPipeVd : Route::kSimtVd, false, nullptr};
  }
  if (g.grad_view_features || g.grad_w3 || g.grad_b3)
    return {Route::kRefused, false,
            "grad_view_features / grad_w3 / grad_b3 need params->view_features"};
  const bool pipe = env && p.workspace_bytes >= (size_t)kWgAccOffset &&
                    (!wgrad || (!g.g_extra &&
                                p.workspace_bytes >= (size_t)NFI_BACKWARD_WORKSPACE_BYTES));
  if (!pipe) return {Route::kSimt, false, nullptr};
  if (!wgrad) return {Route::kPipe, false, nullptr};
  // the generator step (cameras are data) in ONE sweep, with the plane scatter folded into
  // render_wgrad_pipe; with a pose gradient render_backward_pipe runs beside it
  const bool others =
      g.grad_planes || g.grad_palette || g.grad_beta || g.grad_alpha || g.grad_origins;
  if (others && !g.grad_origins && !(p.mlp_mode & kDbgTwoSweeps))
    return {Route::kWgradOneSweep, false, nullptr};
  return {others ? Route::kPipeAndWgrad : Route::kWgrad, false, nullptr};
}

}  // namespace nfi
