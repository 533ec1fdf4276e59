// LPIPS-VGG distance of the inversion loss on sm_90a (C ABI: include/nfi_lpips.h), restating the
// reference's lib/metrics.py:97-137 over lpips.LPIPS(net='vgg').
//
// in0 and in1 run through the network as ONE 2N-image batch (in0 first), channel-last:
//   conv1_1 (3 -> 64)      conv11_forward_kernel, fp32 on the CUDA cores: reads NCHW with the scaling
//                          layer folded in, writes the pre-activation u and relu(u) as the bf16 hi / lo
//                          pair conv1_2 reads (padding 3 channels to a 64-wide tensor-core K block
//                          would cost 20x its 0.057 GFLOP per image)
//   conv1_2 .. conv5_3     conv_tc_kernel of nfi_synth.cu (nfi::synth::conv3x3): TMA ring, bf16-pair
//                          wgmma, epilogue u = acc + bias -> u (fp32), relu(u) -> pair for the next conv
//   max pool 2x2           pool_kernel: max of relu(u) over the window -> pair
//   head (five taps)       head_forward_kernel: per position normalise both images' feature vectors,
//                          sum_c lin[c] (n0 - n1)^2; per (image, 64-position chunk) partial sums in a
//                          fixed order, then head_sum_kernel: out[i] = sum_tap sum_chunk / HW_tap
// No cross-image atomics anywhere: an image's distance and gradient are bit-identical whether it runs
// alone or inside a batch.
//
// Backward to in0 (the first N images; the in1 half of the saved u feeds the head's gradient), or,
// with save = 2 and grad_in1, to both halves as one 2N-image batch (the head is symmetric in the
// pair): walk conv5_3 .. conv1_2 with
//   tap_backward_kernel    g_v = (gradient from the layer above) + (pool adjoint: a scatter to the
//                          window's first maximum, recomputed from the saved u) + (head gradient at a
//                          tap); g_u = g_v relu'(u) -> bf16 pair
//   conv_tc_kernel RAW     the data gradient with the flipped tap table (as the synthesis backward)
//   conv11_backward_kernel relu'(u) and conv1_1's data gradient in fp32, times 1 / scale, += grad_in0
//                          (and grad_in1)
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include "nfi_lpips.h"
#include "nfi_pair.cuh"
#include "nfi_synth_launch.h"

namespace nfi {
namespace lpips {
namespace {

constexpr int kConvs = NFI_LPIPS_CONVS, kTaps = NFI_LPIPS_TAPS;
constexpr int kCin[kConvs] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int kCout[kConvs] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int kLevel[kConvs] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4};  // resolution H >> level
constexpr int kTapOf[kConvs] = {-1, 0, -1, 1, -1, -1, 2, -1, -1, 3, -1, -1, 4};
constexpr int kChunk = 64;        // positions per head partial sum (8 warps x 8 positions)
constexpr float kEps = 1e-10f;    // normalize_tensor

inline bool pooled_after(int l) { return kTapOf[l] >= 0 && l < kConvs - 1; }

// ---------------------------------------------------------------- conv1_1 forward
// One thread per (position, 8 output channels); the 8 threads of a position read the same 27 inputs.
__global__ void __launch_bounds__(256)
conv11_forward_kernel(const float* __restrict__ in0, const float* __restrict__ in1, int N, int H, int W,
                      const float* __restrict__ w, const float* __restrict__ b,
                      const float* __restrict__ shift, const float* __restrict__ scale,
                      float* __restrict__ u, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float ws[27 * 64];  // [ci*9 + tap][co]
  __shared__ float bs[64];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) ws[(i % 27) * 64 + i / 27] = w[i];
  if (threadIdx.x < 64) bs[threadIdx.x] = b[threadIdx.x];
  __syncthreads();
  const size_t HW = (size_t)H * W, total = (size_t)2 * N * HW * 8;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(idx & 7);
    const size_t pos = idx >> 3;
    const int x = (int)(pos % W), y = (int)((pos / W) % H);
    const int img = (int)(pos / HW);
    const float* src = img < N ? in0 + (size_t)img * 3 * HW : in1 + (size_t)(img - N) * 3 * HW;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bs[8 * g + j];
    for (int ci = 0; ci < 3; ++ci) {
      const float sh = shift[ci], sc = scale[ci];
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
        // the conv's zero padding applies to the SCALED image
        const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W)
                            ? (__ldg(src + ci * HW + (size_t)yy * W + xx) - sh) / sc : 0.f;
        const float* wr = ws + (ci * 9 + t) * 64 + 8 * g;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(v, wr[j], acc[j]);
      }
    }
    const size_t o = pos * 64 + 8 * g;
    *reinterpret_cast<float4*>(u + o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(u + o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    __align__(16) __nv_bfloat16 h[8], l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split_bf16(relu(acc[j]), h[j], l[j]);
    *reinterpret_cast<uint4*>(hi + o) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(lo + o) = *reinterpret_cast<const uint4*>(l);
  }
}

// ---------------------------------------------------------------- max pool 2x2
// relu(u) [B,h,w,C] -> max over each 2x2 window -> pair [B,h/2,w/2,C]; one thread per 4 channels
__global__ void __launch_bounds__(256)
pool_kernel(const float* __restrict__ u, int B, int h, int w, int C, __nv_bfloat16* __restrict__ hi,
            __nv_bfloat16* __restrict__ lo) {
  const int oh = h >> 1, ow = w >> 1, c4n = C >> 2;
  const size_t total = (size_t)B * oh * ow * c4n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const size_t op = i / c4n;
    const int ox = (int)(op % ow), oy = (int)((op / ow) % oh);
    const size_t img = op / ((size_t)ow * oh);
    float m[4] = {0.f, 0.f, 0.f, 0.f};  // relu(.) >= 0
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const size_t p = (img * h + 2 * oy + (q >> 1)) * w + 2 * ox + (q & 1);
      const float4 v = __ldg(reinterpret_cast<const float4*>(u + p * C) + c4);
      m[0] = v.x > m[0] ? v.x : m[0];
      m[1] = v.y > m[1] ? v.y : m[1];
      m[2] = v.z > m[2] ? v.z : m[2];
      m[3] = v.w > m[3] ? v.w : m[3];
    }
    __align__(8) __nv_bfloat16 hh[4], ll[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_bf16(m[j], hh[j], ll[j]);
    *reinterpret_cast<uint2*>(hi + op * C + 4 * c4) = *reinterpret_cast<const uint2*>(hh);
    *reinterpret_cast<uint2*>(lo + op * C + 4 * c4) = *reinterpret_cast<const uint2*>(ll);
  }
}

// ---------------------------------------------------------------- head
// Block (chunk, image): 8 warps x 8 positions; a warp holds one position's C channels (KC per lane).
template <int KC>
__global__ void __launch_bounds__(256)
head_forward_kernel(const float* __restrict__ u, int N, int HW, const float* __restrict__ lin,
                    float* __restrict__ partial, int n_chunks) {
  constexpr int C = 32 * KC;
  __shared__ float wsum[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int img = blockIdx.y;
  float wl[KC];
#pragma unroll
  for (int k = 0; k < KC; ++k) wl[k] = __ldg(lin + lane + 32 * k);
  float acc = 0.f;
  for (int j = 0; j < kChunk / 8; ++j) {
    const int p = blockIdx.x * kChunk + warp * (kChunk / 8) + j;
    if (p >= HW) break;
    const float* u0 = u + ((size_t)img * HW + p) * C;
    const float* u1 = u + ((size_t)(N + img) * HW + p) * C;
    float f0[KC], f1[KC], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      f0[k] = relu(__ldg(u0 + lane + 32 * k));
      f1[k] = relu(__ldg(u1 + lane + 32 * k));
      s0 = fmaf(f0[k], f0[k], s0);
      s1 = fmaf(f1[k], f1[k], s1);
    }
    const float e0 = sqrtf(warp_sum(s0)) + kEps, e1 = sqrtf(warp_sum(s1)) + kEps;
    float d = 0.f;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const float t = f0[k] / e0 - f1[k] / e1;
      d = fmaf(wl[k], t * t, d);
    }
    acc += warp_sum(d);
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += wsum[i];
    partial[(size_t)img * n_chunks + blockIdx.x] = s;
  }
}

struct TapOffsets {
  int n_chunks[kTaps];
  int hw[kTaps];
  size_t off[kTaps];  // into the partials
};

// out[i] = sum over taps of (sum over chunks) / HW, in a fixed order (the reference's per-layer
// mean, summed over layers)
__global__ void head_sum_kernel(const float* __restrict__ partial, TapOffsets t, int N, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float d = 0.f;
  for (int l = 0; l < kTaps; ++l) {
    const float* p = partial + t.off[l] + (size_t)i * t.n_chunks[l];
    float s = 0.f;
    for (int c = 0; c < t.n_chunks[l]; ++c) s += p[c];
    d += s / (float)t.hw[l];
  }
  out[i] = d;
}

// ---------------------------------------------------------------- backward
struct TapBackward {
  int N, B, H, W;       // N pairs; B = N (gradient to in0) or 2N (to in0 and in1) images processed
  const float* u;       // [2N,H,W,C] the layer's saved pre-activation (in0's images first)
  const float* g;       // [B,H,W,C] gradient of relu(u) from the conv above, or nullptr
  const float* g_pool;  // [B,H/2,W/2,C] gradient of the pool output above, or nullptr
  const float* lin;     // [C] at a tap, else nullptr
  const float* g_dist;  // [N]
  float inv_hw;
  __nv_bfloat16* hi;    // [B,H,W,C] out: g_u = g_v relu'(u)
  __nv_bfloat16* lo;
};

// One warp per cell: a 2x2 pool window with g_pool, else one position; KC channels per lane.
template <int KC>
__global__ void __launch_bounds__(256)
tap_backward_kernel(TapBackward a) {
  constexpr int C = 32 * KC;
  const int lane = threadIdx.x & 31;
  const bool pool = a.g_pool != nullptr;
  const int cw = pool ? a.W >> 1 : a.W, ch = pool ? a.H >> 1 : a.H;
  const size_t cells = (size_t)a.B * ch * cw, HW = (size_t)a.H * a.W;
  float wl[KC];
#pragma unroll
  for (int k = 0; k < KC; ++k) wl[k] = a.lin ? __ldg(a.lin + lane + 32 * k) : 0.f;
  for (size_t cell = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; cell < cells;
       cell += ((size_t)gridDim.x * blockDim.x) >> 5) {
    const int cx = (int)(cell % cw), cy = (int)((cell / cw) % ch);
    const int img = (int)(cell / ((size_t)cw * ch));
    const int y0 = pool ? 2 * cy : cy, x0 = pool ? 2 * cx : cx;
    // the pool's adjoint: the window's gradient goes to its first maximum in row-major order (as
    // PyTorch's max_pool2d), found again from the saved u
    int am[KC];
    float gp[KC];
#pragma unroll
    for (int k = 0; k < KC; ++k) { am[k] = -1; gp[k] = 0.f; }
    if (pool) {
#pragma unroll
      for (int k = 0; k < KC; ++k) {
        const int c = lane + 32 * k;
        float m = -1.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const size_t p = ((size_t)img * a.H + y0 + (q >> 1)) * a.W + x0 + (q & 1);
          const float v = relu(__ldg(a.u + p * C + c));
          if (v > m) { m = v; am[k] = q; }
        }
        gp[k] = __ldg(a.g_pool + (((size_t)img * ch + cy) * cw + cx) * C + c);
      }
    }
    const bool first = img < a.N;  // in0's image; its partner is in1's, and the other way round
    const float gd = a.lin ? __ldg(a.g_dist + (first ? img : img - a.N)) * a.inv_hw : 0.f;
    for (int q = 0; q < (pool ? 4 : 1); ++q) {
      const size_t pos = ((size_t)img * a.H + y0 + (q >> 1)) * a.W + x0 + (q & 1);
      const float* u0 = a.u + pos * C;
      float f0[KC], gv[KC];
#pragma unroll
      for (int k = 0; k < KC; ++k) {
        f0[k] = __ldg(u0 + lane + 32 * k);
        gv[k] = a.g ? __ldg(a.g + pos * C + lane + 32 * k) : 0.f;
        if (am[k] == q) gv[k] += gp[k];
      }
      if (a.lin) {
        // f0 this image's features, f1 its partner's (the head is symmetric in the two):
        // d/df0 of sum_c lin[c] (f0/(r0+eps) - f1/(r1+eps))^2: with gn = gd 2 lin (n0 - n1),
        // gf = gn/(r0+eps) - f0 (gn . f0) / (r0 (r0+eps)^2); 0 where r0 = 0 (f0 = 0 there)
        const float* u1 = first ? u0 + HW * a.N * C : u0 - HW * a.N * C;
        float f1[KC], s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          const float v = relu(f0[k]);
          f1[k] = relu(__ldg(u1 + lane + 32 * k));
          s0 = fmaf(v, v, s0);
          s1 = fmaf(f1[k], f1[k], s1);
        }
        const float r0 = sqrtf(warp_sum(s0));
        const float e0 = r0 + kEps, e1 = sqrtf(warp_sum(s1)) + kEps;
        float gn[KC], dot = 0.f;
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          const float v = relu(f0[k]);
          gn[k] = gd * 2.f * wl[k] * (v / e0 - f1[k] / e1);
          dot = fmaf(gn[k], v, dot);
        }
        dot = warp_sum(dot);
        if (r0 > 0.f) {
          const float c2 = (dot / r0) / (e0 * e0);   // r0 e0^2 would underflow for r0 < 1e-18
#pragma unroll
          for (int k = 0; k < KC; ++k) gv[k] += gn[k] / e0 - relu(f0[k]) * c2;
        }
      }
#pragma unroll
      for (int k = 0; k < KC; ++k) {
        const size_t o = pos * C + lane + 32 * k;
        split_bf16(f0[k] > 0.f ? gv[k] : 0.f, a.hi[o], a.lo[o]);
      }
    }
  }
}

// grad_in[n,ci,y,x] += sum_{tap,co} relu'(u)[n,y-ky+1,x-kx+1,co] g[..,co] W[co,ci,ky,kx] / scale[ci]:
// one thread per position of the first B images (in0's N, then in1's), into grad_in0 / grad_in1
__global__ void __launch_bounds__(256)
conv11_backward_kernel(const float* __restrict__ g, const float* __restrict__ u, int N, int B, int H, int W,
                       const float* __restrict__ w, const float* __restrict__ scale,
                       float* __restrict__ grad_in0, float* __restrict__ grad_in1) {
  __shared__ float ws[9 * 64 * 3];  // [tap][co][ci]
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) {
    const int co = i / 27, ci = (i / 9) % 3, t = i % 9;
    ws[(t * 64 + co) * 3 + ci] = w[i];
  }
  __syncthreads();
  const size_t HW = (size_t)H * W, total = (size_t)B * HW;
  for (size_t pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x; pos < total;
       pos += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(pos % W), y = (int)((pos / W) % H);
    const size_t img = pos / HW;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int t = 0; t < 9; ++t) {
      const int yy = y - t / 3 + 1, xx = x - t % 3 + 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const size_t q = ((img * H + yy) * W + xx) * 64;
      const float* wt = ws + t * 64 * 3;
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 gv = __ldg(reinterpret_cast<const float4*>(g + q) + c4);
        const float4 uv = __ldg(reinterpret_cast<const float4*>(u + q) + c4);
        const float gu[4] = {uv.x > 0.f ? gv.x : 0.f, uv.y > 0.f ? gv.y : 0.f, uv.z > 0.f ? gv.z : 0.f,
                             uv.w > 0.f ? gv.w : 0.f};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int ci = 0; ci < 3; ++ci) acc[ci] = fmaf(gu[j], wt[(4 * c4 + j) * 3 + ci], acc[ci]);
      }
    }
    float* dst = img < (size_t)N ? grad_in0 + img * 3 * HW : grad_in1 + (img - N) * 3 * HW;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) dst[ci * HW + (size_t)y * W + x] += acc[ci] / scale[ci];
  }
}

// ---------------------------------------------------------------- host side
// The workspace: a deterministic walk, so the backward finds what a saved forward left.
struct Layout {
  Pair wf[kConvs];   // forward weights [9][Cout][Cin] (layers 1..12)
  float* u[kConvs];  // pre-activations [2N,h,w,Cout]: one per layer when saved, else two in turn
  Pair act[2];       // conv inputs [2N,h,w,C], in turn
  float* partial;
  TapOffsets taps;
  // backward (saved only)
  Pair wt[kConvs];   // [9][Cin][Cout]
  float* g[2];       // data gradients [N,h,w,Cin], in turn
  Pair dacc;         // [N,h,w,Cout]
};

static void layout(const nfi_lpips_params& P, Bump& b, Layout& L) {
  const size_t N = P.n, HW = (size_t)P.height * P.width;
  const size_t full = HW * 64;  // the largest per-image tensor of every level (h w C = HW 64 >> level)
  for (int l = 1; l < kConvs; ++l) L.wf[l] = b.pair((size_t)9 * kCin[l] * kCout[l]);
  if (P.save) {
    for (int l = 0; l < kConvs; ++l) L.u[l] = b.take(2 * N * (HW >> (2 * kLevel[l])) * kCout[l]);
  } else {
    float* r[2] = {b.take(2 * N * full), b.take(2 * N * full)};
    for (int l = 0; l < kConvs; ++l) L.u[l] = r[l & 1];
  }
  L.act[0] = b.pair(2 * N * full);
  L.act[1] = b.pair(2 * N * full);
  size_t np = 0;
  for (int t = 0; t < kTaps; ++t) {
    const int hw = (int)(HW >> (2 * t));
    L.taps.hw[t] = hw;
    L.taps.n_chunks[t] = (hw + kChunk - 1) / kChunk;
    L.taps.off[t] = np;
    np += N * L.taps.n_chunks[t];
  }
  L.partial = b.take(np);
  if (P.save) {
    const size_t nb = P.save == 2 ? 2 * N : N;  // images the backward walks: in0's, or both halves
    for (int l = 1; l < kConvs; ++l) L.wt[l] = b.pair((size_t)9 * kCin[l] * kCout[l]);
    L.g[0] = b.take(nb * full);
    L.g[1] = b.take(nb * full);
    L.dacc = b.pair(nb * full);
  }
}

static int check(const nfi_lpips_params& P) {
  if (P.n <= 0) return fail("lpips: N must be positive, got %d", P.n);
  if (P.height < 16 || P.width < 16 || P.height % 16 || P.width % 16)
    return fail("lpips: H and W must be multiples of 16 (four 2x2 pools), got %d x %d", P.height, P.width);
  if (P.save < 0 || P.save > 2) return fail("lpips: save must be 0, 1 or 2, got %d", P.save);
  return 0;
}

template <int KC>
static void head_forward(const float* u, int N, int hw, const float* lin, float* partial, int n_chunks,
                         cudaStream_t st) {
  head_forward_kernel<KC><<<dim3((unsigned)n_chunks, (unsigned)N), 256, 0, st>>>(u, N, hw, lin, partial,
                                                                                 n_chunks);
}
template <int KC>
static void tap_backward(const TapBackward& a, cudaStream_t st) {
  const size_t cells = (size_t)a.B * a.H * a.W / (a.g_pool ? 4 : 1);
  tap_backward_kernel<KC><<<flat_grid(cells * 32), 256, 0, st>>>(a);
}

}  // namespace

size_t workspace_bytes(const nfi_lpips_params& P) {
  if (check(P)) return 0;
  Bump b{nullptr, 0, 0};
  Layout L;
  layout(P, b, L);
  return b.off + 1024;
}

static int setup(const nfi_lpips_params& P, Layout& L) {
  if (const int rc = check(P)) return rc;
  if (!P.in0 || !P.in1 || !P.shift || !P.scale || !P.out || !P.workspace)
    return fail("lpips: in0, in1, shift, scale, out and workspace must be set");
  for (int l = 0; l < kConvs; ++l)
    if (!P.conv_w[l] || !P.conv_b[l]) return fail("lpips: conv %d weight / bias missing", l);
  for (int t = 0; t < kTaps; ++t)
    if (!P.lin_w[t]) return fail("lpips: lin %d missing", t);
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need) return fail("lpips: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  Bump b = aligned_bump(P.workspace, P.workspace_bytes);
  layout(P, b, L);
  return 0;
}

int forward(const nfi_lpips_params& P, cudaStream_t st) {
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const int N = P.n, H = P.height, W = P.width, B2 = 2 * N;
  for (int l = 1; l < kConvs; ++l)
    if (const int rc = synth::prep_weights(P.conv_w[l], kCout[l], kCin[l], 9, 9 * kCin[l], 1.f, synth::kTapCoCi,
                                           L.wf[l], st))
      return rc;
  conv11_forward_kernel<<<flat_grid((size_t)B2 * H * W * 8), 256, 0, st>>>(
      P.in0, P.in1, N, H, W, P.conv_w[0], P.conv_b[0], P.shift, P.scale, L.u[0], L.act[0].hi, L.act[0].lo);
  NFI_CUDA(cudaGetLastError());
  int cur = 0;
  for (int l = 1; l < kConvs; ++l) {
    const int h = H >> kLevel[l], w = W >> kLevel[l], t = kTapOf[l];
    const bool writes_pair = t < 0;  // a tap's relu(u) is read from u (head, pool)
    const Pair out = writes_pair ? L.act[cur ^ 1] : Pair{nullptr, nullptr};
    if (const int rc = synth::conv3x3(B2, h, w, kCin[l], kCout[l], L.act[cur], L.wf[l], P.conv_b[l], L.u[l], out, st))
      return rc;
    if (t >= 0) {
      float* part = L.partial + L.taps.off[t];
      const int hw = h * w, nc = L.taps.n_chunks[t];
      switch (kCout[l]) {
        case 64: head_forward<2>(L.u[l], N, hw, P.lin_w[t], part, nc, st); break;
        case 128: head_forward<4>(L.u[l], N, hw, P.lin_w[t], part, nc, st); break;
        case 256: head_forward<8>(L.u[l], N, hw, P.lin_w[t], part, nc, st); break;
        default: head_forward<16>(L.u[l], N, hw, P.lin_w[t], part, nc, st); break;
      }
      NFI_CUDA(cudaGetLastError());
      if (pooled_after(l)) {
        pool_kernel<<<flat_grid((size_t)B2 * (h / 2) * (w / 2) * (kCout[l] / 4)), 256, 0, st>>>(
            L.u[l], B2, h, w, kCout[l], L.act[cur ^ 1].hi, L.act[cur ^ 1].lo);
        NFI_CUDA(cudaGetLastError());
      }
    }
    cur ^= 1;
  }
  head_sum_kernel<<<(N + 255) / 256, 256, 0, st>>>(L.partial, L.taps, N, P.out);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int backward(const nfi_lpips_params& P, const float* g_dist, float* grad_in0, float* grad_in1, cudaStream_t st) {
  if (!P.save || (grad_in1 && P.save != 2))
    return fail("lpips backward: needs the workspace of a forward with save = 1 (save = 2 "
                "for a gradient to in1)");
  if (!g_dist || !grad_in0) return fail("lpips backward: g_dist and grad_in0 must be set");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const int N = P.n, H = P.height, W = P.width, B = grad_in1 ? 2 * N : N;
  for (int l = 1; l < kConvs; ++l)
    if (const int rc = synth::prep_weights(P.conv_w[l], kCout[l], kCin[l], 9, 9 * kCin[l], 1.f, synth::kTapCiCo,
                                           L.wt[l], st))
      return rc;
  const float* gin = nullptr;  // gradient of layer l's relu(u), or of the pool output after it
  int cur = 0;
  for (int l = kConvs - 1; l >= 1; --l) {
    const int h = H >> kLevel[l], w = W >> kLevel[l], t = kTapOf[l];
    TapBackward a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.B = B; a.H = h; a.W = w; a.u = L.u[l];
    if (pooled_after(l)) a.g_pool = gin; else a.g = gin;
    if (t >= 0) { a.lin = P.lin_w[t]; a.g_dist = g_dist; a.inv_hw = 1.f / (float)(h * w); }
    a.hi = L.dacc.hi; a.lo = L.dacc.lo;
    switch (kCout[l]) {
      case 64: tap_backward<2>(a, st); break;
      case 128: tap_backward<4>(a, st); break;
      case 256: tap_backward<8>(a, st); break;
      default: tap_backward<16>(a, st); break;
    }
    NFI_CUDA(cudaGetLastError());
    if (const int rc = synth::conv3x3_adjoint(B, h, w, kCout[l], kCin[l], L.dacc, L.wt[l], L.g[cur], st))
      return rc;
    gin = L.g[cur];
    cur ^= 1;
  }
  conv11_backward_kernel<<<flat_grid((size_t)B * H * W), 256, 0, st>>>(gin, L.u[0], N, B, H, W, P.conv_w[0],
                                                                      P.scale, grad_in0, grad_in1);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int saved_preactivation(const nfi_lpips_params& P, int layer, float* out, cudaStream_t st) {
  if (!P.save || layer < 0 || layer >= kConvs || out == nullptr)
    return fail("lpips saved_preactivation: needs a saved forward, a layer in 0..12, out");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const size_t n = (size_t)2 * P.n * ((size_t)P.height * P.width >> (2 * kLevel[layer])) * kCout[layer];
  NFI_CUDA(cudaMemcpyAsync(out, L.u[layer], n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // namespace lpips
}  // namespace nfi

using nfi::fail;

extern "C" {

size_t nfi_lpips_workspace_bytes(const nfi_lpips_params* params) {
  if (params == nullptr) return 0;
  return nfi::lpips::workspace_bytes(*params);
}

int nfi_lpips_forward(const nfi_lpips_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::lpips::forward(*params, (cudaStream_t)stream);
}

int nfi_lpips_backward(const nfi_lpips_params* params, const float* g_dist, float* grad_in0, float* grad_in1,
                       void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::lpips::backward(*params, g_dist, grad_in0, grad_in1, (cudaStream_t)stream);
}

int nfi_lpips_saved_preactivation(const nfi_lpips_params* params, int32_t layer, float* out, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::lpips::saved_preactivation(*params, layer, out, (cudaStream_t)stream);
}

}  // extern "C"
