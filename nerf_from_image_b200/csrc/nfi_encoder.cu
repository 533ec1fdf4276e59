// Regression heads of the bootstrap encoder on sm_90a (C ABI: include/nfi_encoder.h), restating the
// reference's models/encoder.py:70-103 from the backbone output(s) on.
//
// Forward, channel-last throughout (M = B 4h 4w image positions):
//   synth::transpose       features [B,C,h,w] -> fp32 [B,h,w,C]
//   upsample_relu_kernel   relu(bilinear x4, align_corners=False, PyTorch's scale_factor index rule)
//                          -> x0 pair [M,C], the A operand of the first conv; at scale 1 the same
//                          kernel writes relu(features_latent) -> xl pair [B,h,w,C]
//   conv_tc_kernel         post[0], post[2] (nfi::synth::conv3x3): bias, ReLU -> a1, a2 pairs;
//                          post[4] with Cout zero-padded 4 -> 32 (the kernel's narrowest N):
//                          pre-activation -> maps_kernel -> maps [M,4]; w_regressor_pre[0] at h x w:
//                          pre-activation ul [B,h,w,C]
//   mean_pool_kernel       pooled[b,c] = sum_p relu(ul) / (h w), per image in a fixed order
//
// Backward (every sum over positions or images in a fixed order; no atomics):
//   act_backward_kernel    g_maps -> a 64-channel zero-padded pair (TMA needs 16-byte rows), the
//                          adjoint conv's input and the weight GEMM's G; between convs the RAW data
//                          gradient times relu' (from the saved pair's sign) -> pair; the mean pool's
//                          adjoint g_pooled / (h w) relu'(ul) -> pair.  Each writes per-chunk
//                          partial sums of its gradient; synth::bias_reduce adds them to the bias
//                          gradient in chunk order
//   conv_tc_kernel RAW     the data gradients with the flipped tap table (nfi::synth::conv3x3_adjoint)
//   wgrad_tc_kernel        the weight gradients (nfi::synth::wgrad3x3): G against the saved input
//   upsample_adjoint_kernel each source texel gathers the destination pixels whose bilinear footprint
//                          covers it (clamped borders included), times relu' of the upsample; at
//                          scale 1 it is relu'(features_latent) times the gradient; synth::transpose
//                          adds the result into g_features / g_features_latent ([B,C,h,w])
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <limits.h>
#include <string.h>

#include "nfi_encoder.h"
#include "nfi_pair.cuh"
#include "nfi_synth_launch.h"

namespace nfi {
namespace encoder {
namespace {

constexpr int kScale = 4;     // SegFormer's output is 1/4 of the image (encoder.py:75-80)
constexpr int kMaps = NFI_ENCODER_MAPS;
constexpr int kMapsN = 32;    // post[4]'s Cout on conv_tc_kernel (its narrowest N)
constexpr int kMapsG = 64;    // g_maps' channels as a pair (one 64-channel K block, 128-byte rows)
constexpr int kRows = 256;    // positions per partial bias sum

// relu(bilinear upsample by S) of f [B,h,w,C] -> pair [B,Sh,Sw,C]; one thread per 4 channels
__global__ void __launch_bounds__(256)
upsample_relu_kernel(const float* __restrict__ f, int B, int h, int w, int C, int S,
                     __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int Ho = S * h, Wo = S * w, c4n = C >> 2;
  const float inv_s = 1.f / (float)S;
  const size_t total = (size_t)B * Ho * Wo * c4n;
  const float4* f4 = reinterpret_cast<const float4*>(f);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const size_t p = i / c4n;
    const int X = (int)(p % Wo), Y = (int)((p / Wo) % Ho);
    const size_t b = p / ((size_t)Wo * Ho);
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    src_index(Y, inv_s, h, y0, y1, ly0, ly1);
    src_index(X, inv_s, w, x0, x1, lx0, lx1);
    const float4 v00 = __ldg(f4 + ((b * h + y0) * w + x0) * c4n + c4);
    const float4 v01 = __ldg(f4 + ((b * h + y0) * w + x1) * c4n + c4);
    const float4 v10 = __ldg(f4 + ((b * h + y1) * w + x0) * c4n + c4);
    const float4 v11 = __ldg(f4 + ((b * h + y1) * w + x1) * c4n + c4);
    const float v[4] = {ly0 * (lx0 * v00.x + lx1 * v01.x) + ly1 * (lx0 * v10.x + lx1 * v11.x),
                        ly0 * (lx0 * v00.y + lx1 * v01.y) + ly1 * (lx0 * v10.y + lx1 * v11.y),
                        ly0 * (lx0 * v00.z + lx1 * v01.z) + ly1 * (lx0 * v10.z + lx1 * v11.z),
                        ly0 * (lx0 * v00.w + lx1 * v01.w) + ly1 * (lx0 * v10.w + lx1 * v11.w)};
    __align__(8) __nv_bfloat16 hh[4], ll[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_bf16(relu(v[j]), hh[j], ll[j]);
    *reinterpret_cast<uint2*>(hi + i * 4) = *reinterpret_cast<const uint2*>(hh);
    *reinterpret_cast<uint2*>(lo + i * 4) = *reinterpret_cast<const uint2*>(ll);
  }
}

// The adjoint of upsample_relu_kernel: out[b,i,j,c] = sum over destination pixels (Y,X) of
// wy(Y -> i) wx(X -> j) d[b,Y,X,c] [mask_hi[b,Y,X,c] > 0]; the candidates are Y in
// [S(i-1), S(i+2)) (the taps of every destination row lie within one source row of it)
__global__ void __launch_bounds__(256)
upsample_adjoint_kernel(const float* __restrict__ d, const __nv_bfloat16* __restrict__ mask_hi, int B,
                        int h, int w, int C, int S, float* __restrict__ out) {
  const int Ho = S * h, Wo = S * w, c4n = C >> 2;
  const float inv_s = 1.f / (float)S;
  const size_t total = (size_t)B * h * w * c4n;
  const float4* d4 = reinterpret_cast<const float4*>(d);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const size_t p = i / c4n;
    const int sj = (int)(p % w), si = (int)((p / w) % h);
    const size_t b = p / ((size_t)w * h);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int ya = max(0, S * (si - 1)), yb = min(Ho, S * (si + 2));
    const int xa = max(0, S * (sj - 1)), xb = min(Wo, S * (sj + 2));
    for (int Y = ya; Y < yb; ++Y) {
      const float wy = src_weight(Y, si, inv_s, h);
      if (wy == 0.f) continue;
      for (int X = xa; X < xb; ++X) {
        const float wx = src_weight(X, sj, inv_s, w);
        if (wx == 0.f) continue;
        const float wt = wy * wx;
        const size_t q = ((b * Ho + Y) * Wo + X) * c4n + c4;
        const float4 g = __ldg(d4 + q);
        const uint2 mb = __ldg(reinterpret_cast<const uint2*>(mask_hi) + q);
        const __nv_bfloat16* m = reinterpret_cast<const __nv_bfloat16*>(&mb);
        if (__bfloat162float(m[0]) > 0.f) acc.x += wt * g.x;
        if (__bfloat162float(m[1]) > 0.f) acc.y += wt * g.y;
        if (__bfloat162float(m[2]) > 0.f) acc.z += wt * g.z;
        if (__bfloat162float(m[3]) > 0.f) acc.w += wt * g.w;
      }
    }
    reinterpret_cast<float4*>(out)[i] = acc;
  }
}

// post[4]'s pre-activation u [M,32] -> maps [M,4]
__global__ void __launch_bounds__(256)
maps_kernel(const float* __restrict__ u, size_t M, float* __restrict__ maps) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (size_t)gridDim.x * blockDim.x)
    reinterpret_cast<float4*>(maps)[i] = __ldg(reinterpret_cast<const float4*>(u + i * kMapsN));
}

// pooled[b,c] = sum_p relu(u[b,p,c]) / HW.  Block (64-channel chunk, image): 4 row groups of 64
// channels, each summing every fourth position in order, then combined in a fixed order.
__global__ void __launch_bounds__(256)
mean_pool_kernel(const float* __restrict__ u, int HW, int C, float* __restrict__ pooled) {
  __shared__ float part[4][64];
  const int c = blockIdx.x * 64 + (threadIdx.x & 63), g = threadIdx.x >> 6;
  const size_t b = blockIdx.y;
  float s = 0.f;
  for (int p = g; p < HW; p += 4) s += relu(__ldg(u + (b * HW + p) * C + c));
  part[g][threadIdx.x & 63] = s;
  __syncthreads();
  if (g == 0) {
    const int k = threadIdx.x;
    pooled[b * C + c] = (((part[0][k] + part[1][k]) + part[2][k]) + part[3][k]) / (float)HW;
  }
}

struct ActBackward {
  int M, C, out_C;               // positions; gradient channels; pair channels (>= C, rest zero)
  const float* g;                // [M,C] gradient, or nullptr: the broadcast form below
  const float* g_img;            // [M / per_img, C] times g_scale at every position of the image
  int per_img;
  float g_scale;
  const __nv_bfloat16* mask_hi;  // [M,C] the branch: pass where the saved activation is > 0
  const float* mask_u;           // [M,C] or: pass where the saved pre-activation is > 0
  __nv_bfloat16* hi;             // [M,out_C] out
  __nv_bfloat16* lo;
  float* partial;                // [chunks][C] sums over the chunk's kRows positions, in order
};

// One block per chunk of kRows positions, one thread per channel (coalesced rows)
__global__ void __launch_bounds__(256)
act_backward_kernel(const ActBackward a) {
  const int r0 = blockIdx.x * kRows, r1 = min(a.M, r0 + kRows);
  for (int c = threadIdx.x; c < a.out_C; c += blockDim.x) {
    float s = 0.f;
    for (int r = r0; r < r1; ++r) {
      float v = 0.f;
      if (c < a.C) {
        const size_t o = (size_t)r * a.C + c;
        v = a.g ? __ldg(a.g + o) : __ldg(a.g_img + (size_t)(r / a.per_img) * a.C + c) * a.g_scale;
        if (a.mask_hi && !(__bfloat162float(a.mask_hi[o]) > 0.f)) v = 0.f;
        if (a.mask_u && !(__ldg(a.mask_u + o) > 0.f)) v = 0.f;
        s += v;
      }
      const size_t q = (size_t)r * a.out_C + c;
      split_bf16(v, a.hi[q], a.lo[q]);
    }
    if (c < a.C) a.partial[(size_t)blockIdx.x * a.C + c] = s;
  }
}

// a saved activation as fp32: hi + lo of a pair, or relu(u)
__global__ void __launch_bounds__(256)
unpack_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
              const float* __restrict__ u, size_t n, float* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = u ? relu(u[i]) : __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}

// ---------------------------------------------------------------- host side
// The workspace: a deterministic walk, so the backward finds what a saved forward left.
struct Layout {
  float* fcl;          // [B,h,w,C] a backbone output channel-last (also the backward's gather out)
  // pose head
  Pair w0, w2, w4;     // forward weights [9][Cout][Cin] (w4: Cout padded to 32)
  float* w4p;          // post[4]'s weight [64,C,3,3] and bias [64], zero-padded
  float* b4p;
  Pair x0, a1, a2;     // [M,C] (a2 shares x0's storage without save)
  float* u4;           // [M,32]
  // latent head
  Pair wl;
  Pair xl;             // [B,h,w,C]
  float* ul;           // [B,h,w,C]
  // backward (save only)
  Pair t0, t2, t4, tl; // [9][Cin][Cout] (t4: Cout padded to 64)
  Pair g4;             // [M,64]
  float* d;            // [M,C] (pose) or [B,h,w,C] data gradient
  Pair g;              // [M,C] or [B,h,w,C] gradient pair
  float* part;         // the weight GEMM's partial sums, the largest of the layers'
  float* bpart;        // partial bias sums
};

static void layout(const nfi_encoder_params& P, Bump& b, Layout& L) {
  memset(&L, 0, sizeof(L));
  const size_t B = P.batch, C = P.channels, hw = (size_t)P.height * P.width;
  const size_t M = B * hw * kScale * kScale, Ml = B * hw;
  const int H = kScale * P.height, W = kScale * P.width;
  const size_t wsz = (size_t)9 * C * C;
  L.fcl = b.take(Ml * C);
  size_t part = 0, bchunks = 0;
  if (P.pose_regressor) {
    L.w0 = b.pair(wsz);
    L.w2 = b.pair(wsz);
    L.w4 = b.pair((size_t)9 * kMapsN * C);
    L.w4p = b.take((size_t)kMapsG * C * 9);
    L.b4p = b.take(kMapsG);
    L.x0 = b.pair(M * C);
    L.a1 = b.pair(M * C);
    L.a2 = P.save ? b.pair(M * C) : L.x0;
    L.u4 = b.take(M * kMapsN);
    const size_t pc = synth::wgrad3x3_partial_floats(P.batch, H, W, P.channels, P.channels);
    const size_t p4 = synth::wgrad3x3_partial_floats(P.batch, H, W, kMaps, P.channels);
    part = pc > p4 ? pc : p4;
    bchunks = blocks(M, kRows);
  }
  if (P.latent_regressor) {
    L.wl = b.pair(wsz);
    L.xl = b.pair(Ml * C);
    L.ul = b.take(Ml * C);
    const size_t pl = synth::wgrad3x3_partial_floats(P.batch, P.height, P.width, P.channels, P.channels);
    part = part > pl ? part : pl;
    bchunks = bchunks > blocks(Ml, kRows) ? bchunks : blocks(Ml, kRows);
  }
  if (P.save) {
    const size_t big = P.pose_regressor ? M : Ml;
    if (P.pose_regressor) {
      L.t0 = b.pair(wsz);
      L.t2 = b.pair(wsz);
      L.t4 = b.pair((size_t)9 * C * kMapsG);
      L.g4 = b.pair(M * kMapsG);
    }
    if (P.latent_regressor) L.tl = b.pair(wsz);
    L.d = b.take(big * C);
    L.g = b.pair(big * C);
    L.part = b.take(part);
    L.bpart = b.take(bchunks * C);
  }
}

static int check(const nfi_encoder_params& P) {
  if (P.batch <= 0 || P.batch > 65535 || P.height <= 0 || P.width <= 0 || P.height > 1024 ||
      P.width > 1024)
    return fail("encoder: B in 1..65535 and feature sizes in 1..1024 needed, got B %d, %d x %d",
                P.batch, P.height, P.width);
  if ((size_t)P.batch * kScale * kScale * P.height * P.width > (size_t)INT_MAX)
    return fail("encoder: more than 2^31 image positions (B %d, %d x %d features)", P.batch, P.height, P.width);
  if (P.channels <= 0 || P.channels % 64 != 0)
    return fail("encoder: channels must be a positive multiple of 64, got %d", P.channels);
  if ((P.pose_regressor != 0 && P.pose_regressor != 1) || (P.latent_regressor != 0 && P.latent_regressor != 1) ||
      !(P.pose_regressor || P.latent_regressor))
    return fail("encoder: pose_regressor and latent_regressor are 0 or 1, and one is 1");
  if (P.save != 0 && P.save != 1) return fail("encoder: save must be 0 or 1, got %d", P.save);
  return 0;
}

// the pair of a gradient with relu' applied, and its sum over positions into g_b (if set)
static int act_backward(ActBackward a, float* g_b, cudaStream_t st) {
  const int n = (int)blocks((size_t)a.M, kRows);
  act_backward_kernel<<<n, 256, 0, st>>>(a);
  NFI_CUDA(cudaGetLastError());
  return synth::bias_reduce(a.partial, n, a.C, g_b, st);
}

}  // namespace

size_t workspace_bytes(const nfi_encoder_params& P) {
  if (check(P)) return 0;
  Bump b{nullptr, 0, 0};
  Layout L;
  layout(P, b, L);
  return b.off + 1024;
}

static int setup(const nfi_encoder_params& P, Layout& L) {
  if (const int rc = check(P)) return rc;
  if (P.pose_regressor && (!P.features || !P.post0_w || !P.post0_b || !P.post2_w || !P.post2_b || !P.post4_w ||
                           !P.post4_b || !P.maps))
    return fail("encoder: the pose head needs features, post weights and biases, and maps");
  if (P.latent_regressor && (!P.features_latent || !P.wpre_w || !P.wpre_b || !P.pooled))
    return fail("encoder: the latent head needs features_latent, w_regressor_pre's weight and "
                "bias, and pooled");
  if (!P.workspace) return fail("encoder: workspace missing");
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need) return fail("encoder: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  Bump b = aligned_bump(P.workspace, P.workspace_bytes);
  layout(P, b, L);
  return 0;
}

int forward(const nfi_encoder_params& P, cudaStream_t st) {
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const int B = P.batch, h = P.height, w = P.width, C = P.channels, H = kScale * h, W = kScale * w;
  const size_t M = (size_t)B * H * W, Ml = (size_t)B * h * w;
  const Pair none = {nullptr, nullptr};
  if (P.pose_regressor) {
    NFI_CUDA(cudaMemsetAsync(L.w4p, 0, (size_t)kMapsG * C * 9 * sizeof(float), st));
    NFI_CUDA(cudaMemsetAsync(L.b4p, 0, kMapsG * sizeof(float), st));
    NFI_CUDA(
cudaMemcpyAsync(L.w4p, P.post4_w, (size_t)kMaps * C * 9 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    NFI_CUDA(cudaMemcpyAsync(L.b4p, P.post4_b, kMaps * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (int rc = synth::prep_weights(P.post0_w, C, C, 9, 9 * C, 1.f, synth::kTapCoCi, L.w0, st))
      return rc;
    if (int rc = synth::prep_weights(P.post2_w, C, C, 9, 9 * C, 1.f, synth::kTapCoCi, L.w2, st))
      return rc;
    if (int rc = synth::prep_weights(L.w4p, kMapsN, C, 9, 9 * C, 1.f, synth::kTapCoCi, L.w4, st))
      return rc;
    if (int rc = synth::transpose(P.features, B, C, h * w, nullptr, 0, L.fcl, st)) return rc;
    upsample_relu_kernel<<<flat_grid(M * C / 4), 256, 0, st>>>(L.fcl, B, h, w, C, kScale, L.x0.hi, L.x0.lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv3x3(B, H, W, C, C, L.x0, L.w0, P.post0_b, nullptr, L.a1, st)) return rc;
    if (int rc = synth::conv3x3(B, H, W, C, C, L.a1, L.w2, P.post2_b, nullptr, L.a2, st)) return rc;
    if (int rc = synth::conv3x3(B, H, W, C, kMapsN, L.a2, L.w4, L.b4p, L.u4, none, st)) return rc;
    maps_kernel<<<flat_grid(M), 256, 0, st>>>(L.u4, M, P.maps);
    NFI_CUDA(cudaGetLastError());
  }
  if (P.latent_regressor) {
    if (int rc = synth::prep_weights(P.wpre_w, C, C, 9, 9 * C, 1.f, synth::kTapCoCi, L.wl, st)) return rc;
    if (int rc = synth::transpose(P.features_latent, B, C, h * w, nullptr, 0, L.fcl, st)) return rc;
    upsample_relu_kernel<<<flat_grid(Ml * C / 4), 256, 0, st>>>(L.fcl, B, h, w, C, 1, L.xl.hi, L.xl.lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv3x3(B, h, w, C, C, L.xl, L.wl, P.wpre_b, L.ul, none, st)) return rc;
    mean_pool_kernel<<<dim3((unsigned)(C / 64), (unsigned)B), 256, 0, st>>>(L.ul, h * w, C, P.pooled);
    NFI_CUDA(cudaGetLastError());
  }
  return 0;
}

int backward(const nfi_encoder_params& P, const float* g_maps, const float* g_pooled, const nfi_encoder_grads& G,
             cudaStream_t st) {
  if (!P.save) return fail("encoder backward: needs the workspace of a forward with save = 1");
  if ((P.pose_regressor && !g_maps) || (P.latent_regressor && !g_pooled))
    return fail("encoder backward: g_maps (pose head) and g_pooled (latent head) must be set");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const int B = P.batch, h = P.height, w = P.width, C = P.channels, H = kScale * h, W = kScale * w;
  const int M = B * H * W, Ml = B * h * w;
  if (P.pose_regressor) {
    if (int rc = synth::prep_weights(P.post0_w, C, C, 9, 9 * C, 1.f, synth::kTapCiCo, L.t0, st))
      return rc;
    if (int rc = synth::prep_weights(P.post2_w, C, C, 9, 9 * C, 1.f, synth::kTapCiCo, L.t2, st))
      return rc;
    if (int rc = synth::prep_weights(L.w4p, kMapsG, C, 9, 9 * C, 1.f, synth::kTapCiCo, L.t4, st))
      return rc;
    ActBackward a;
    memset(&a, 0, sizeof(a));
    a.M = M; a.partial = L.bpart;
    // post[4]: g_maps as the zero-padded pair
    a.C = kMaps; a.out_C = kMapsG; a.g = g_maps; a.hi = L.g4.hi; a.lo = L.g4.lo;
    if (int rc = act_backward(a, G.g_post4_b, st)) return rc;
    if (int rc = synth::wgrad3x3(B, H, W, kMaps, C, kMapsG, L.g4, L.a2, L.part, G.g_post4_w, st))
      return rc;
    const bool below2 = G.g_post2_w || G.g_post2_b || G.g_post0_w || G.g_post0_b || G.g_features;
    const bool below0 = G.g_post0_w || G.g_post0_b || G.g_features;
    if (below2) {
      if (int rc = synth::conv3x3_adjoint(B, H, W, kMapsG, C, L.g4, L.t4, L.d, st)) return rc;
      // post[2]
      a.C = C; a.out_C = C; a.g = L.d; a.mask_hi = L.a2.hi; a.hi = L.g.hi; a.lo = L.g.lo;
      if (int rc = act_backward(a, G.g_post2_b, st)) return rc;
      if (int rc = synth::wgrad3x3(B, H, W, C, C, C, L.g, L.a1, L.part, G.g_post2_w, st))
        return rc;
    }
    if (below0) {
      if (int rc = synth::conv3x3_adjoint(B, H, W, C, C, L.g, L.t2, L.d, st)) return rc;
      // post[0]
      a.mask_hi = L.a1.hi;
      if (int rc = act_backward(a, G.g_post0_b, st)) return rc;
      if (int rc = synth::wgrad3x3(B, H, W, C, C, C, L.g, L.x0, L.part, G.g_post0_w, st))
        return rc;
    }
    if (G.g_features) {
      if (int rc = synth::conv3x3_adjoint(B, H, W, C, C, L.g, L.t0, L.d, st)) return rc;
      upsample_adjoint_kernel<<<flat_grid((size_t)Ml * C / 4), 256, 0, st>>>(L.d, L.x0.hi, B, h, w, C, kScale,
                                                                             L.fcl);
      NFI_CUDA(cudaGetLastError());
      if (int rc = synth::transpose(L.fcl, B, h * w, C, nullptr, 1, G.g_features, st)) return rc;
    }
  }
  if (P.latent_regressor) {
    if (int rc = synth::prep_weights(P.wpre_w, C, C, 9, 9 * C, 1.f, synth::kTapCiCo, L.tl, st)) return rc;
    ActBackward a;
    memset(&a, 0, sizeof(a));
    a.M = Ml; a.C = C; a.out_C = C; a.partial = L.bpart;
    a.g_img = g_pooled; a.per_img = h * w; a.g_scale = 1.f / (float)(h * w);
    a.mask_u = L.ul; a.hi = L.g.hi; a.lo = L.g.lo;
    if (int rc = act_backward(a, G.g_wpre_b, st)) return rc;
    if (int rc = synth::wgrad3x3(B, h, w, C, C, C, L.g, L.xl, L.part, G.g_wpre_w, st))
      return rc;
    if (G.g_features_latent) {
      if (int rc = synth::conv3x3_adjoint(B, h, w, C, C, L.g, L.tl, L.d, st)) return rc;
      upsample_adjoint_kernel<<<flat_grid((size_t)Ml * C / 4), 256, 0, st>>>(L.d, L.xl.hi, B, h, w, C, 1, L.fcl);
      NFI_CUDA(cudaGetLastError());
      if (int rc = synth::transpose(L.fcl, B, h * w, C, nullptr, 1, G.g_features_latent, st))
        return rc;
    }
  }
  return 0;
}

int saved_activation(const nfi_encoder_params& P, int layer, float* out, cudaStream_t st) {
  if (!P.save || layer < 0 || layer > 4 || out == nullptr || (layer < 3 && !P.pose_regressor) ||
      (layer >= 3 && !P.latent_regressor))
    return fail("encoder saved_activation: needs a saved forward, a layer in 0..4 of a head it "
                "ran, out");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const size_t C = P.channels, hw = (size_t)P.height * P.width, n = (size_t)P.batch * hw * C;
  const Pair src[4] = {L.x0, L.a1, L.a2, L.xl};
  const size_t count = layer < 3 ? n * kScale * kScale : n;
  if (layer == 4)
    unpack_kernel<<<flat_grid(count), 256, 0, st>>>(nullptr, nullptr, L.ul, count, out);
  else
    unpack_kernel<<<flat_grid(count), 256, 0, st>>>(src[layer].hi, src[layer].lo, nullptr, count, out);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace encoder
}  // namespace nfi

using nfi::fail;

extern "C" {

size_t nfi_encoder_workspace_bytes(const nfi_encoder_params* params) {
  if (params == nullptr) return 0;
  return nfi::encoder::workspace_bytes(*params);
}

int nfi_encoder_forward(const nfi_encoder_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::encoder::forward(*params, (cudaStream_t)stream);
}

int nfi_encoder_backward(const nfi_encoder_params* params, const float* g_maps, const float* g_pooled,
                         const nfi_encoder_grads* grads, void* stream) {
  if (params == nullptr || grads == nullptr) return fail("params / grads is NULL");
  return nfi::encoder::backward(*params, g_maps, g_pooled, *grads, (cudaStream_t)stream);
}

int nfi_encoder_saved_activation(const nfi_encoder_params* params, int32_t layer, float* out, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::encoder::saved_activation(*params, layer, out, (cudaStream_t)stream);
}

}  // extern "C"
