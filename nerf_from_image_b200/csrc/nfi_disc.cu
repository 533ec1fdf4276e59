// The GAN discriminator's backbone on sm_90a (C ABI: include/nfi_disc.h), restating the
// reference's models/stylegan.py:493-676 from the image and the conditioning map on.
//
// Forward, channel-last throughout; block i runs at r = R >> i with C -> C' channels, h = r / 2:
//   fromrgb_kernel      img [B,nc,R,R] -> x pair [B,R,R,C]: 1x1 in fp32, bias, lrelu sqrt2
//   conv_tc_kernel      conv0 (nfi::synth::conv3x3_act): bias, lrelu sqrt2 -> a pair
//   fir_phases_kernel   filter2d^T(a) (4x4 [1,3,3,1]^2/64, pad 1: [B,r+1,r+1,C]) as its four parity
//                       phases [4B,h+1,h+1,C] (pair)
//   conv_tc_kernel      conv1 as 9 stride-1 taps over the phases (nfi::synth::conv_down3x3) -> raw
//   fir_down_kernel     downsample2d(x) (the same filter, stride 2, pad 1) -> pair [B,h,h,C]
//   conv_tc_kernel      skip 1x1 (nfi::synth::conv1x1), gain sqrt2/2 folded into the weights -> raw
//   block_out_kernel    u1 = raw1 + b1 (saved), x' = lrelu(u1) + skip -> the next block's pair, or
//                       fp32 [B,4,4,512] after the last block
//   4x4, in fp32 on the CUDA cores: mbstd_kernel (concat -> [B,16,513]), b4_conv_kernel (-> u, a in
//   flatten order [B,512*16]), linear_kernel (fc with lrelu sqrt2; out), logits_kernel
//
// Backward (every sum over positions or images in a fixed order; no atomics), one reverse walk that
// the R1 double backward below also runs, over a stacked [g; g-dot]:
//   epilogue_backward, 4x4: logits_backward_kernel, linear_dx / linear_dw kernels, b4_conv_dx / _dw
//   kernels, mbstd_backward_kernel -> g of the last block's output, fp32 [B,4,4,512]
//   reverse_walk, per block from the last to the first, over the walk's 1 or 2 copies of B images:
//     out_backward_kernel  g_y -> pairs of g_y (the skip's output gradient) and g_u1 = g_y lrelu'(u1)
//                          (conv1's), with per-chunk sums of g_u1 for the bias; once per copy
//     wgrad_tc_kernel      conv1 (transposed, against the phases), skip (against the downsampled x)
//     conv_tc_kernel RAW   conv1's data gradient: the stride-2 transposed conv (conv_up3x3) ->
//                          [B,r+1,r+1,C]; skip's (conv1x1 with transposed weights) -> [B,h,h,C]
//     fir_up_act_kernel    the adjoint of filter2d^T, times sqrt2 lrelu'(conv0) -> pair, bias sums;
//                          once per copy
//     wgrad_tc_kernel      conv0;  conv_tc_kernel RAW: its data gradient (flipped taps) -> g_x
//     fir_down_adjoint_kernel  g_x += downsample2d^T(skip's data gradient)
//   then fromrgb_backward_kernel / fromrgb_gimg_kernel: the 1x1 in fp32 (weight, bias, image gradients)
// Each weight gradient sums its terms (one here, two in R1) in a scratch buffer and
// synth::wgrad_terms adds gain x it (transposed for conv1) to the caller's.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "nfi_disc.h"
#include "nfi_disc_r1.h"
#include "nfi_pair.cuh"
#include "nfi_synth_launch.h"

namespace nfi {
namespace disc {
namespace {

constexpr int kMaxBlocks = NFI_DISC_MAX_BLOCKS;
constexpr int kC4 = 512;        // channels at 4x4 (channel_max)
constexpr int kCat = kC4 + 1;   // with the minibatch-std channel
constexpr int kFcIn = kC4 * 16;
constexpr int kGroup = 4;       // minibatch-std group (stylegan.py:577)
constexpr int kRows = 256;      // positions per partial bias sum
constexpr int kLinImg = 8;      // images per linear_kernel block
constexpr float kSlope = 0.2f;
constexpr float kSqrt2 = 1.41421356237309505f;

// [1,3,3,1] / 8 per axis: bilinear_filter() is its outer product, normalised to sum 1
__device__ __forceinline__ float fir(int u) { return (u == 0 || u == 3) ? 0.125f : 0.375f; }
__device__ __forceinline__ float pair_at(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t i) {
  return __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
// lrelu' on the branch a saved activation pair took (its hi half has the sign)
__device__ __forceinline__ float branch(const __nv_bfloat16* hi, size_t i) {
  return __bfloat162float(hi[i]) > 0.f ? 1.f : kSlope;
}

// Minibatch-std group j (images j + k B/4, k < 4) at element e of [16,512]: the values v, their
// mean m, var = sum_k (v_k - m)^2 and s = sqrt(var / 4 + 1e-8); along a tangent dx also its values
// dv, their mean dm and dvar = sum_k (v_k - m)(dv_k - dm).
struct Group {
  float v[kGroup], m, var, s;
  float dv[kGroup], dm, dvar;
};
__device__ __forceinline__ Group group(const float* __restrict__ x, int G, int j, int e) {
  Group q;
  q.m = 0.f;
  for (int k = 0; k < kGroup; ++k) {
    q.v[k] = __ldg(x + (size_t)(k * G + j) * 16 * kC4 + e);
    q.m += q.v[k];
  }
  q.m /= (float)kGroup;
  q.var = 0.f;
  for (int k = 0; k < kGroup; ++k) q.var += (q.v[k] - q.m) * (q.v[k] - q.m);
  q.s = sqrtf(q.var / (float)kGroup + 1e-8f);
  return q;
}
__device__ __forceinline__ Group group(const float* __restrict__ x, const float* __restrict__ dx, int G, int j,
                                       int e) {
  Group q = group(x, G, j, e);
  q.dm = 0.f;
  for (int k = 0; k < kGroup; ++k) {
    q.dv[k] = __ldg(dx + (size_t)(k * G + j) * 16 * kC4 + e);
    q.dm += q.dv[k];
  }
  q.dm /= (float)kGroup;
  q.dvar = 0.f;
  for (int k = 0; k < kGroup; ++k) q.dvar += (q.v[k] - q.m) * (q.dv[k] - q.dm);
  return q;
}
// G_j: the std channel's gradient in g_xs [B,16,513], summed over group j's images and positions
__device__ __forceinline__ float std_grad_sum(const float* __restrict__ gxs, int G, int j) {
  float gs = 0.f;
  for (int k = 0; k < kGroup; ++k)
    for (int p = 0; p < 16; ++p) gs += __ldg(gxs + ((size_t)(k * G + j) * 16 + p) * kCat + kC4);
  return gs;
}

int channels(int r) { return r >= 64 ? 32768 / r > 512 ? 512 : 32768 / r : 512; }
int n_blocks(int R) {
  int n = 0;
  for (int r = R; r > 4; r >>= 1) ++n;
  return n;
}

// the 4x4 conv's weights [512][513][9] * gain -> fp32 [513*9][512]
__global__ void w4_kernel(const float* __restrict__ w, float gain, float* __restrict__ wt) {
  const size_t n = (size_t)kC4 * kCat * 9;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int co = (int)(i / (kCat * 9)), k = (int)(i % (kCat * 9));
    wt[(size_t)k * kC4 + co] = w[i] * gain;
  }
}

// x[b,p,c] = lrelu(sqrt2 (sum_ci (w[c,ci] g) img[b,ci,p] + bias[c])) -> pair [B,R,R,C]
__global__ void __launch_bounds__(256)
fromrgb_kernel(const float* __restrict__ img, int B, int nc, int RR, int C, const float* __restrict__ w,
               float g, const float* __restrict__ bias, __nv_bfloat16* __restrict__ hi,
               __nv_bfloat16* __restrict__ lo) {
  const size_t total = (size_t)B * RR * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t q = i / C;
    const int p = (int)(q % RR);
    const size_t b = q / RR;
    float s = 0.f;
    for (int ci = 0; ci < nc; ++ci) s += (__ldg(w + c * nc + ci) * g) * __ldg(img + (b * nc + ci) * RR + p);
    split_bf16(lrelu((s + __ldg(bias + c)) * kSqrt2, kSlope), hi[i], lo[i]);
  }
}

// f = filter2d^T(a) on [B,r,r,C] (f[o] = sum_u fir(u) a[o-2+u], o in 0..r) as phases
// P[(2py+px) B + b, m, n] = f[2m+py, 2n+px], m, n in 0..h (zero beyond r)
__global__ void __launch_bounds__(256)
fir_phases_kernel(const __nv_bfloat16* __restrict__ ahi, const __nv_bfloat16* __restrict__ alo, int B, int r,
                  int C, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int h1 = r / 2 + 1;
  const size_t total = (size_t)4 * B * h1 * h1 * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t q = i / C;
    const int n = (int)(q % h1);
    q /= h1;
    const int m = (int)(q % h1);
    q /= h1;
    const int b = (int)(q % B), ph = (int)(q / B);
    const int oy = 2 * m + (ph >> 1), ox = 2 * n + (ph & 1);
    float s = 0.f;
    if (oy <= r && ox <= r) {
      for (int u = 0; u < 4; ++u) {
        const int y = oy - 2 + u;
        if (y < 0 || y >= r) continue;
        float sr = 0.f;
        for (int v = 0; v < 4; ++v) {
          const int x = ox - 2 + v;
          if (x < 0 || x >= r) continue;
          sr += fir(v) * pair_at(ahi, alo, (((size_t)b * r + y) * r + x) * C + c);
        }
        s += fir(u) * sr;
      }
    }
    split_bf16(s, hi[i], lo[i]);
  }
}

// downsample2d: d[i,j] = sum_{u,v} fir(u) fir(v) x[2i+u-1, 2j+v-1] on [B,r,r,C] -> pair [B,h,h,C]
__global__ void __launch_bounds__(256)
fir_down_kernel(const __nv_bfloat16* __restrict__ xhi, const __nv_bfloat16* __restrict__ xlo, int B, int r,
                int C, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int h = r / 2;
  const size_t total = (size_t)B * h * h * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t q = i / C;
    const int j = (int)(q % h);
    q /= h;
    const int ii = (int)(q % h);
    const size_t b = q / h;
    float s = 0.f;
    for (int u = 0; u < 4; ++u) {
      const int y = 2 * ii + u - 1;
      if (y < 0 || y >= r) continue;
      float sr = 0.f;
      for (int v = 0; v < 4; ++v) {
        const int x = 2 * j + v - 1;
        if (x < 0 || x >= r) continue;
        sr += fir(v) * pair_at(xhi, xlo, ((b * r + y) * r + x) * C + c);
      }
      s += fir(u) * sr;
    }
    split_bf16(s, hi[i], lo[i]);
  }
}

// u1 = raw1 + b1 -> u_out; y = lrelu(u1) + skip -> pair and / or fp32
__global__ void __launch_bounds__(256)
block_out_kernel(const float* __restrict__ raw1, const float* __restrict__ skip, const float* __restrict__ b1,
                 size_t n, int C, float* __restrict__ u_out, __nv_bfloat16* __restrict__ hi,
                 __nv_bfloat16* __restrict__ lo, float* __restrict__ y_out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float u = __ldg(raw1 + i) + __ldg(b1 + i % C);
    u_out[i] = u;
    const float y = __ldg(skip + i) + lrelu(u, kSlope);
    if (hi != nullptr) split_bf16(y, hi[i], lo[i]);
    if (y_out != nullptr) y_out[i] = y;
  }
}

// Minibatch std: group j holds images j + k B/4 (k < 4).  One block per group: sd[j] = mean over
// (p, c) of sqrt(var_k + 1e-8), summed per thread then in a fixed tree; xs [B,16,513] = x and sd.
__global__ void __launch_bounds__(256)
mbstd_kernel(const float* __restrict__ x, int B, float* __restrict__ xs, float* __restrict__ sd) {
  __shared__ float part[256];
  const int G = B / kGroup, j = blockIdx.x;
  float s = 0.f;
  for (int e = threadIdx.x; e < 16 * kC4; e += 256) {
    const Group q = group(x, G, j, e);
    s += q.s;
    for (int k = 0; k < kGroup; ++k) xs[((size_t)(k * G + j) * 16 + e / kC4) * kCat + e % kC4] = q.v[k];
  }
  part[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < kGroup * 16) {
    const int k = threadIdx.x / 16, p = threadIdx.x % 16;
    xs[((size_t)(k * G + j) * 16 + p) * kCat + kC4] = part[0] / (float)(16 * kC4);
  }
  if (threadIdx.x == 0) sd[j] = part[0] / (float)(16 * kC4);
}

// The 4x4 conv, 513 -> 512, pad 1: block (image, 64 outputs), thread (co, 4 positions); the
// image in shared memory, weights wt [513*9][512] (gain folded).  u = sqrt2 (conv + b) and
// lrelu(u), both in flatten order [B][512*16] (index co*16 + p).
__global__ void __launch_bounds__(256)
b4_conv_kernel(const float* __restrict__ xs, const float* __restrict__ wt, const float* __restrict__ bias,
               float* __restrict__ u, float* __restrict__ a) {
  __shared__ float sx[16 * kCat];
  const size_t b = blockIdx.x;
  for (int i = threadIdx.x; i < 16 * kCat; i += 256) sx[i] = __ldg(xs + b * 16 * kCat + i);
  __syncthreads();
  const int co = blockIdx.y * 64 + (threadIdx.x & 63), p0 = (threadIdx.x >> 6) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ci = 0; ci < kCat; ++ci)
    for (int t = 0; t < 9; ++t) {
      const float w = __ldg(wt + ((size_t)ci * 9 + t) * kC4 + co);
      const int dy = t / 3 - 1, dx = t % 3 - 1;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int y = (p0 + q) / 4 + dy, x = (p0 + q) % 4 + dx;
        if (y >= 0 && y < 4 && x >= 0 && x < 4) acc[q] += w * sx[(y * 4 + x) * kCat + ci];
      }
    }
  for (int q = 0; q < 4; ++q) {
    const float v = (acc[q] + __ldg(bias + co)) * kSqrt2;
    const size_t o = b * kFcIn + (size_t)co * 16 + p0 + q;
    u[o] = v;
    a[o] = lrelu(v, kSlope);
  }
}

// y[b,o] = (sum_k (W[o,k] g) x[b,k] + bias[o]) (* sqrt2, lrelu with act).  Block (o, 8 images):
// each thread sums every 256th k, then a fixed tree per image.
__global__ void __launch_bounds__(256)
linear_kernel(const float* __restrict__ x, const float* __restrict__ W, float g, const float* __restrict__ bias,
              int B, int K, int O, int act, float* __restrict__ u, float* __restrict__ y) {
  __shared__ float part[kLinImg][256];
  const int o = blockIdx.x, b0 = blockIdx.y * kLinImg;
  float s[kLinImg];
  for (int q = 0; q < kLinImg; ++q) s[q] = 0.f;
  for (int k = threadIdx.x; k < K; k += 256) {
    const float w = __ldg(W + (size_t)o * K + k) * g;
    for (int q = 0; q < kLinImg; ++q)
      if (b0 + q < B) s[q] += w * __ldg(x + (size_t)(b0 + q) * K + k);
  }
  for (int q = 0; q < kLinImg; ++q) part[q][threadIdx.x] = s[q];
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int q = 0; q < kLinImg; ++q) part[q][threadIdx.x] += part[q][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < kLinImg && b0 + (int)threadIdx.x < B) {
    const int b = b0 + threadIdx.x;
    float v = part[threadIdx.x][0] + __ldg(bias + o);
    if (act) v *= kSqrt2;
    if (u != nullptr) u[(size_t)b * O + o] = v;
    y[(size_t)b * O + o] = act ? lrelu(v, kSlope) : v;
  }
}

// logits[b] = sum_c out[b,c] cmap[b,c] / sqrt(D), or out[b,0] without a map
__global__ void logits_kernel(const float* __restrict__ out, const float* __restrict__ cmap, int B, int D,
                              float* __restrict__ logits) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (D == 0) {
    logits[b] = out[b];
    return;
  }
  float s = 0.f;
  for (int c = 0; c < D; ++c) s += out[(size_t)b * D + c] * cmap[(size_t)b * D + c];
  logits[b] = s / sqrtf((float)D);
}

// g_out[b,c] = g[b] cmap[b,c] / sqrt(D) (g[b] without a map); g_cmap[b,c] += g[b] out[b,c] / sqrt(D)
__global__ void logits_backward_kernel(const float* __restrict__ g, const float* __restrict__ out,
                                       const float* __restrict__ cmap, int B, int D, float* __restrict__ g_out,
                                       float* __restrict__ g_cmap) {
  const int N = D ? D : 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * N) return;
  const int b = i / N;
  if (D == 0) {
    g_out[i] = g[b];
    return;
  }
  const float s = 1.f / sqrtf((float)D);
  g_out[i] = g[b] * cmap[i] * s;
  if (g_cmap != nullptr) g_cmap[i] += g[b] * out[i] * s;
}

// g_u = g_y gain lrelu'(u); runs in place (gu == gy), so neither is __restrict__
__global__ void act_backward_kernel(const float* gy, const float* __restrict__ u, size_t n, float gain, float* gu) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    gu[i] = gy[i] * gain * lrelu_grad(u[i], kSlope);
}

// g_x[b,k] = sum_o g_u[b,o] W[o,k] g
__global__ void linear_dx_kernel(const float* __restrict__ gu, const float* __restrict__ W, float g, int B, int K,
                                 int O, float* __restrict__ gx) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * K) return;
  const int k = (int)(i % K);
  const size_t b = i / K;
  float s = 0.f;
  for (int o = 0; o < O; ++o) s += __ldg(gu + b * O + o) * (__ldg(W + (size_t)o * K + k) * g);
  gx[i] = s;
}

// g_W[o,k] += g sum_b g_u[b,o] x[b,k]; g_bias[o] += sum_b g_u[b,o] (from the k = 0 thread)
__global__ void linear_dw_kernel(const float* __restrict__ gu, const float* __restrict__ x, float g, int B, int K,
                                 int O, float* __restrict__ gW, float* __restrict__ gb) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)O * K) return;
  const int k = (int)(i % K), o = (int)(i / K);
  if (gW != nullptr) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += __ldg(gu + (size_t)b * O + o) * __ldg(x + (size_t)b * K + k);
    gW[i] += g * s;
  }
  if (gb != nullptr && k == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += __ldg(gu + (size_t)b * O + o);
    gb[o] += s;
  }
}

// The 4x4 conv's data gradient: g_xs[b,p,ci] = sum_{co,tap} g_u[b,co,p - tap] W[co,ci,tap] g.
// Thread (image, ci), all 16 positions; g_u of the image in shared memory.
__global__ void __launch_bounds__(256)
b4_conv_dx_kernel(const float* __restrict__ gu, const float* __restrict__ W, float g, float* __restrict__ gxs) {
  __shared__ float sg[kFcIn];
  const size_t b = blockIdx.y;
  for (int i = threadIdx.x; i < kFcIn; i += 256) sg[i] = __ldg(gu + b * kFcIn + i);
  __syncthreads();
  const int ci = blockIdx.x * 256 + threadIdx.x;
  if (ci >= kCat) return;
  float acc[16];
  for (int p = 0; p < 16; ++p) acc[p] = 0.f;
  for (int co = 0; co < kC4; ++co) {
    float w[9];
    for (int t = 0; t < 9; ++t) w[t] = __ldg(W + ((size_t)co * kCat + ci) * 9 + t) * g;
    // input position p = (y, x) feeds output (y - dy, x - dx) through tap (dy + 1, dx + 1)
    for (int p = 0; p < 16; ++p) {
      const int y = p / 4, x = p % 4;
      float s = 0.f;
      for (int t = 0; t < 9; ++t) {
        const int oy = y - (t / 3 - 1), ox = x - (t % 3 - 1);
        if (oy >= 0 && oy < 4 && ox >= 0 && ox < 4) s += w[t] * sg[co * 16 + oy * 4 + ox];
      }
      acc[p] += s;
    }
  }
  for (int p = 0; p < 16; ++p) gxs[(b * 16 + p) * kCat + ci] = acc[p];
}

// The 4x4 conv's weight gradient, thread per (co, ci, tap): g_W += g sum_{b,p} g_u[b,co,p] xs[b,p+tap,ci];
// the tap-0, ci-0 thread also adds the bias gradient sum_{b,p} g_u[b,co,p]
__global__ void b4_conv_dw_kernel(const float* __restrict__ gu, const float* __restrict__ xs, float g, int B,
                                  float* __restrict__ gW, float* __restrict__ gb) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)kC4 * kCat * 9) return;
  const int t = (int)(i % 9), ci = (int)((i / 9) % kCat), co = (int)(i / (9 * kCat));
  const int dy = t / 3 - 1, dx = t % 3 - 1;
  if (gW != nullptr) {
    float s = 0.f;
    for (int b = 0; b < B; ++b)
      for (int p = 0; p < 16; ++p) {
        const int y = p / 4 + dy, x = p % 4 + dx;
        if (y < 0 || y >= 4 || x < 0 || x >= 4) continue;
        s += __ldg(gu + (size_t)b * kFcIn + co * 16 + p) * __ldg(xs + ((size_t)b * 16 + y * 4 + x) * kCat + ci);
      }
    gW[i] += g * s;
  }
  if (gb != nullptr && t == 0 && ci == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b)
      for (int p = 0; p < 16; ++p) s += __ldg(gu + (size_t)b * kFcIn + co * 16 + p);
    gb[co] += s;
  }
}

// The minibatch std's adjoint: g_x = g_xs[..512] + G_j / (16 * 512) (x_k - m) / (4 s), with G_j the
// sum of the std channel's gradient over the group's images and positions.  Thread per (group, e).
__global__ void mbstd_backward_kernel(const float* __restrict__ gxs, const float* __restrict__ x, int B,
                                      float* __restrict__ gx) {
  const int G = B / kGroup;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * 16 * kC4) return;
  const int e = (int)(i % (16 * kC4)), j = (int)(i / (16 * kC4));
  const float gs = std_grad_sum(gxs, G, j);
  const Group q = group(x, G, j, e);
  const float c = gs / (float)(16 * kC4) / ((float)kGroup * q.s);
  for (int k = 0; k < kGroup; ++k) {
    const size_t b = (size_t)(k * G + j);
    gx[b * 16 * kC4 + e] = __ldg(gxs + (b * 16 + e / kC4) * kCat + e % kC4) + c * (q.v[k] - q.m);
  }
}

// g_y of a block [M,C]: pairs of g_y (skip) and g_u1 = g_y lrelu'(u1) (conv1), and per-chunk sums of
// g_u1 over kRows positions.  One block per chunk, one thread per channel.
__global__ void __launch_bounds__(256)
out_backward_kernel(const float* __restrict__ gy, const float* __restrict__ u1, int M, int C,
                    __nv_bfloat16* __restrict__ yhi, __nv_bfloat16* __restrict__ ylo,
                    __nv_bfloat16* __restrict__ uhi, __nv_bfloat16* __restrict__ ulo, float* __restrict__ partial) {
  const int r0 = blockIdx.x * kRows, r1 = min(M, r0 + kRows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int r = r0; r < r1; ++r) {
      const size_t o = (size_t)r * C + c;
      const float g = __ldg(gy + o), gu = g * lrelu_grad(__ldg(u1 + o), kSlope);
      split_bf16(g, yhi[o], ylo[o]);
      split_bf16(gu, uhi[o], ulo[o]);
      s += gu;
    }
    partial[(size_t)blockIdx.x * C + c] = s;
  }
}

// The adjoint of filter2d^T: g_a[p] = sum_{u,v} fir(u) fir(v) g_f[py+2-u, px+2-v] (g_f [B,r+1,r+1,C]),
// then g_u0 = g_a sqrt2 lrelu'(a) -> pair, with per-chunk sums.  One block per chunk of positions.
__global__ void __launch_bounds__(256)
fir_up_act_kernel(const float* __restrict__ gf, const __nv_bfloat16* __restrict__ ahi, int B, int r, int C,
                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, float* __restrict__ partial) {
  const int M = B * r * r, r1n = r + 1;
  const int p0 = blockIdx.x * kRows, p1 = min(M, p0 + kRows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int q = p0; q < p1; ++q) {
      const int x = q % r, y = (q / r) % r, b = q / (r * r);
      float acc = 0.f;
      for (int u = 0; u < 4; ++u) {
        const int fy = y + 2 - u;
        if (fy < 0 || fy > r) continue;
        float ar = 0.f;
        for (int v = 0; v < 4; ++v) {
          const int fx = x + 2 - v;
          if (fx < 0 || fx > r) continue;
          ar += fir(v) * __ldg(gf + (((size_t)b * r1n + fy) * r1n + fx) * C + c);
        }
        acc += fir(u) * ar;
      }
      const size_t o = (size_t)q * C + c;
      const float g = acc * kSqrt2 * branch(ahi, o);
      split_bf16(g, hi[o], lo[o]);
      s += g;
    }
    partial[(size_t)blockIdx.x * C + c] = s;
  }
}

// g_x[b,y,x] += sum over (i,j,u,v) with 2i+u-1 = y, 2j+v-1 = x of fir(u) fir(v) g_d[b,i,j]
__global__ void __launch_bounds__(256)
fir_down_adjoint_kernel(const float* __restrict__ gd, int B, int r, int C, float* __restrict__ gx) {
  const int h = r / 2;
  const size_t total = (size_t)B * r * r * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t q = i / C;
    const int x = (int)(q % r);
    q /= r;
    const int y = (int)(q % r);
    const size_t b = q / r;
    float s = 0.f;
    for (int u = 0; u < 4; ++u) {
      if ((y + 1 - u) & 1) continue;
      const int ii = (y + 1 - u) / 2;
      if (y + 1 - u < 0 || ii >= h) continue;
      float sr = 0.f;
      for (int v = 0; v < 4; ++v) {
        if ((x + 1 - v) & 1) continue;
        const int jj = (x + 1 - v) / 2;
        if (x + 1 - v < 0 || jj >= h) continue;
        sr += fir(v) * __ldg(gd + ((b * h + ii) * h + jj) * C + c);
      }
      s += fir(u) * sr;
    }
    gx[i] += s;
  }
}

// fromrgb's weight and bias gradients: g_u = g_x sqrt2 lrelu'(x); per chunk of positions and channel
// c, partial[chunk][c][0] = sum g_u, [1 + ci] = sum g_u img[ci].  One thread per channel.
__global__ void __launch_bounds__(256)
fromrgb_backward_kernel(const float* __restrict__ gx, const __nv_bfloat16* __restrict__ xhi,
                        const float* __restrict__ img, int B, int nc, int RR, int C, float* __restrict__ partial) {
  const int M = B * RR;
  const int r0 = blockIdx.x * kRows, r1 = min(M, r0 + kRows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    for (int q = r0; q < r1; ++q) {
      const size_t o = (size_t)q * C + c;
      const float g = __ldg(gx + o) * kSqrt2 * branch(xhi, o);
      const int b = q / RR, p = q % RR;
      s[0] += g;
      for (int ci = 0; ci < nc; ++ci) s[1 + ci] += g * __ldg(img + ((size_t)b * nc + ci) * RR + p);
    }
    for (int k = 0; k <= nc; ++k) partial[((size_t)blockIdx.x * C + c) * (1 + nc) + k] = s[k];
  }
}

__global__ void fromrgb_reduce_kernel(const float* __restrict__ partial, int chunks, int C, int nc, float g,
                                      float* __restrict__ gw, float* __restrict__ gb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * (1 + nc)) return;
  const int c = i / (1 + nc), k = i % (1 + nc);
  float s = 0.f;
  for (int ch = 0; ch < chunks; ++ch) s += partial[((size_t)ch * C + c) * (1 + nc) + k];
  if (k == 0) {
    if (gb != nullptr) gb[c] += s;
  } else if (gw != nullptr) {
    gw[c * nc + k - 1] += g * s;
  }
}

// g_img[b,ci,p] += sum_c (w[c,ci] g) g_x[b,p,c] sqrt2 lrelu'(x).  One warp per position: the lanes
// read the position's channels coalesced, each sums every 32nd channel, then a fixed xor tree.
__global__ void __launch_bounds__(256)
fromrgb_gimg_kernel(const float* __restrict__ gx, const __nv_bfloat16* __restrict__ xhi,
                    const float* __restrict__ w, float g, int B, int nc, int RR, int C, float* __restrict__ gimg) {
  const size_t M = (size_t)B * RR;
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t q = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < M; q += warps) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = lane; c < C; c += 32) {
      const size_t o = q * C + c;
      const float gu = __ldg(gx + o) * kSqrt2 * branch(xhi, o);
      for (int ci = 0; ci < nc; ++ci) s[ci] += (__ldg(w + c * nc + ci) * g) * gu;
    }
#pragma unroll
    for (int ci = 0; ci < 4; ++ci)
      for (int off = 16; off > 0; off >>= 1) s[ci] += __shfl_xor_sync(0xffffffffu, s[ci], off);
    if (lane == 0) {
      const size_t b = q / RR, p = q % RR;
      for (int ci = 0; ci < nc; ++ci) gimg[(b * nc + ci) * RR + p] += s[ci];
    }
  }
}

// a saved tensor as fp32: hi + lo of a pair, or a copy
__global__ void __launch_bounds__(256)
unpack_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
              const float* __restrict__ u, size_t n, float* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = u ? u[i] : __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}

// ---------------------------------------------------------------- host side
struct BlockShape {
  int r, h, C, Co;
};
static BlockShape shape(int R, int i) {
  BlockShape s;
  s.r = R >> i;
  s.h = s.r / 2;
  s.C = channels(s.r);
  s.Co = channels(s.h);
  return s;
}

// The largest per-block sizes (floats or pair elements), which the buffers reused block by block take
struct Sizes {
  size_t big;   // [B,r,r,C]
  size_t bigo;  // [B,h,h,C']
  size_t bigf;  // [B,r+1,r+1,C]
  size_t bigw;  // a 3x3 weight, 9 C max(C, C')
  size_t part;  // weight-GEMM partials
  size_t bp;    // partial sums of the bias and fromrgb reductions
};

static Sizes sizes(const nfi_disc_params& P) {
  Sizes z = {};
  const size_t B = P.batch;
  for (int i = 0; i < n_blocks(P.resolution); ++i) {
    const BlockShape s = shape(P.resolution, i);
    const size_t rr = (size_t)s.r * s.r, hh = (size_t)s.h * s.h;
    z.big = std::max(z.big, B * rr * s.C);
    z.bigo = std::max(z.bigo, B * hh * s.Co);
    z.bigf = std::max(z.bigf, B * (s.r + 1) * (s.r + 1) * s.C);
    z.bigw = std::max(z.bigw, (size_t)9 * s.C * std::max(s.C, s.Co));
    z.part = std::max({z.part, synth::wgrad3x3_partial_floats(P.batch, s.r, s.r, s.C, s.C),
                       synth::wgrad_down3x3_partial_floats(P.batch, s.h, s.C, s.Co),
                       synth::wgrad1x1_partial_floats(P.batch, s.h, s.Co, s.C)});
    z.bp = std::max({z.bp, (size_t)blocks(B * rr, kRows) * s.C * (i == 0 ? 1 + P.img_channels : 1),
                     (size_t)blocks(B * hh, kRows) * s.Co});
  }
  return z;
}

// The reverse walk's buffers, for `copies` stacked copies of the B images: the first-order backward
// walks g (one copy), the HVP [g; g-dot] (two).
struct Reverse {
  Pair t0, t1, ts;       // transposed weights
  float* gA;             // fp32 gradients, largest [copies B,r,r,C]
  float* gB;
  float* gf;             // [copies B,r+1,r+1,C]
  float* gd;             // [copies B,h,h,C]
  Pair gy, gu;           // [copies B,h,h,C'] pairs
  Pair g0;               // [copies B,r,r,C] pair
  float* part;           // weight-GEMM partials
  float* wtmp;           // weight gradient before its gain
  float* bpart;          // partial sums
  float* g4[4];          // 4x4 epilogue gradients (g only): [B,N], [B,512], [B,8192], [B,16,513]
};

static void reverse_layout(const nfi_disc_params& P, const Sizes& z, int copies, Bump& b, Reverse& V) {
  const size_t B = P.batch, n = copies, N = P.cmap_dim ? P.cmap_dim : 1;
  V.t0 = b.pair(z.bigw);
  V.t1 = b.pair(z.bigw);
  V.ts = b.pair(z.bigw / 9);
  V.gA = b.take(n * z.big);
  V.gB = b.take(n * z.big);
  V.gf = b.take(n * z.bigf);
  V.gd = b.take(n * z.bigo);
  V.gy = b.pair(n * z.bigo);
  V.gu = b.pair(n * z.bigo);
  V.g0 = b.pair(n * z.big);
  V.part = b.take(z.part);
  V.wtmp = b.take(z.bigw);
  V.bpart = b.take(z.bp);
  V.g4[0] = b.take(B * N);
  V.g4[1] = b.take(B * kC4);
  V.g4[2] = b.take(B * kFcIn);
  V.g4[3] = b.take(B * 16 * kCat);
}

// The workspace: a deterministic walk, so the backward finds what a saved forward left.
struct Layout {
  Pair x[kMaxBlocks];    // block input [B,r,r,C] (x[0]: fromrgb's output)
  Pair a[kMaxBlocks];    // conv0 output [B,r,r,C]
  Pair ph[kMaxBlocks];   // filter2d^T(a) as phases [4B,h+1,h+1,C]
  Pair d[kMaxBlocks];    // downsample2d(x) [B,h,h,C]
  float* u1[kMaxBlocks]; // conv1 pre-activation [B,h,h,C']
  Pair w0, w1, ws;       // forward weights of one block at a time
  float* raw1;           // [B,h,h,C'] largest
  float* raws;
  float* x4;             // [B,16,512] the last block's output
  float* xs;             // [B,16,513]
  float* sd;             // [B/4]
  float* wt4;            // [513*9][512]
  float* u4;             // [B,8192]
  float* a4;
  float* uf;             // [B,512]
  float* hf;
  float* out;            // [B,N]
  Reverse rev;           // the first-order backward's (save only)
};

static void layout(const nfi_disc_params& P, Bump& b, Layout& L) {
  memset(&L, 0, sizeof(L));
  const Sizes z = sizes(P);
  const size_t B = P.batch, N = P.cmap_dim ? P.cmap_dim : 1;
  for (int i = 0; i < n_blocks(P.resolution); ++i) {
    const BlockShape s = shape(P.resolution, i);
    const size_t rr = (size_t)s.r * s.r, hh = (size_t)s.h * s.h;
    L.x[i] = b.pair(B * rr * s.C);
    L.a[i] = b.pair(B * rr * s.C);
    L.ph[i] = b.pair(4 * B * (s.h + 1) * (s.h + 1) * s.C);
    L.d[i] = b.pair(B * hh * s.C);
    L.u1[i] = b.take(B * hh * s.Co);
  }
  L.w0 = b.pair(z.bigw);
  L.w1 = b.pair(z.bigw);
  L.ws = b.pair(z.bigw / 9);
  L.raw1 = b.take(z.bigo);
  L.raws = b.take(z.bigo);
  L.x4 = b.take(B * kFcIn);
  L.xs = b.take(B * 16 * kCat);
  L.sd = b.take(B / kGroup);
  L.wt4 = b.take((size_t)kCat * 9 * kC4);
  L.u4 = b.take(B * kFcIn);
  L.a4 = b.take(B * kFcIn);
  L.uf = b.take(B * kC4);
  L.hf = b.take(B * kC4);
  L.out = b.take(B * N);
  if (P.save) reverse_layout(P, z, 1, b, L.rev);
}

static int check(const nfi_disc_params& P) {
  const int R = P.resolution;
  if (P.batch <= 0 || P.batch % kGroup != 0 || P.batch > 4096)
    return fail("discriminator: B must be a positive multiple of 4 up to 4096, got %d", P.batch);
  if (R < 8 || R > 256 || (R & (R - 1)) != 0)
    return fail("discriminator: resolution must be a power of two in 8..256, got %d", R);
  if (P.img_channels < 1 || P.img_channels > 4)
    return fail("discriminator: img_channels must be in 1..4, got %d", P.img_channels);
  if (P.cmap_dim != 0 && P.cmap_dim != kC4) return fail("discriminator: cmap_dim must be 0 or 512, got %d", P.cmap_dim);
  if (P.save != 0 && P.save != 1) return fail("discriminator: save must be 0 or 1, got %d", P.save);
  return 0;
}

size_t workspace_bytes(const nfi_disc_params& P) {
  if (check(P)) return 0;
  Bump b{nullptr, 0, 0};
  Layout L;
  layout(P, b, L);
  return b.off + 1024;
}

static int setup(const nfi_disc_params& P, Layout& L) {
  if (const int rc = check(P)) return rc;
  const int nb = n_blocks(P.resolution);
  bool ok = P.img && P.fromrgb_w && P.fromrgb_b && P.b4_conv_w && P.b4_conv_b && P.fc_w && P.fc_b && P.out_w &&
            P.out_b && P.logits && (P.cmap_dim == 0 || P.cmap);
  for (int i = 0; i < nb; ++i)
    ok = ok && P.conv0_w[i] && P.conv0_b[i] && P.conv1_w[i] && P.conv1_b[i] && P.skip_w[i];
  if (!ok)
    return fail("discriminator: img, every weight and bias of the %d blocks and the 4x4 "
                "epilogue, logits, and cmap (with cmap_dim 512) are needed", nb);
  if (!P.workspace) return fail("discriminator: workspace missing");
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need)
    return fail("discriminator: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  Bump b = aligned_bump(P.workspace, P.workspace_bytes);
  layout(P, b, L);
  return 0;
}

static float conv_gain(int cin, int k) { return 1.f / sqrtf((float)(cin * k * k)); }
static const float kSkipGain = 0.70710678118654752f;  // sqrt2 / 2

Pair shifted(Pair p, size_t n) { return Pair{p.hi + n, p.lo + n}; }

// The 4x4 epilogue's backward: g_logits -> g of the last block's output in V.gA [B,16,512].  The out,
// fc and conv weight gradients pair g with hf, a4 and xs: the saved forward's, or in the HVP their
// tangents, where the bias gradients are zero and not asked for.
static int epilogue_backward(const nfi_disc_params& P, const Layout& L, const Reverse& V, const float* g_logits,
                             const float* hf, const float* a4, const float* xs, float* gw_out, float* gw_fc,
                             float* gw_b4, float* gb_out, float* gb_fc, float* gb_b4, float* grad_cmap,
                             cudaStream_t st) {
  const int B = P.batch, N = P.cmap_dim ? P.cmap_dim : 1;
  float *g_out = V.g4[0], *g_hf = V.g4[1], *g_a4 = V.g4[2], *g_xs = V.g4[3];
  logits_backward_kernel<<<blocks((size_t)B * N, 256), 256, 0, st>>>(g_logits, L.out, P.cmap, B, P.cmap_dim,
                                                                     g_out, grad_cmap);
  NFI_CUDA(cudaGetLastError());
  const float g_out_w = 1.f / sqrtf((float)kC4), g_fc_w = 1.f / sqrtf((float)kFcIn);
  linear_dw_kernel<<<blocks((size_t)N * kC4, 256), 256, 0, st>>>(g_out, hf, g_out_w, B, kC4, N, gw_out, gb_out);
  NFI_CUDA(cudaGetLastError());
  linear_dx_kernel<<<blocks((size_t)B * kC4, 256), 256, 0, st>>>(g_out, P.out_w, g_out_w, B, kC4, N, g_hf);
  NFI_CUDA(cudaGetLastError());
  act_backward_kernel<<<flat_grid((size_t)B * kC4), 256, 0, st>>>(g_hf, L.uf, (size_t)B * kC4, kSqrt2, g_hf);
  NFI_CUDA(cudaGetLastError());
  linear_dw_kernel<<<blocks((size_t)kC4 * kFcIn, 256), 256, 0, st>>>(g_hf, a4, g_fc_w, B, kFcIn, kC4, gw_fc, gb_fc);
  NFI_CUDA(cudaGetLastError());
  linear_dx_kernel<<<blocks((size_t)B * kFcIn, 256), 256, 0, st>>>(g_hf, P.fc_w, g_fc_w, B, kFcIn, kC4, g_a4);
  NFI_CUDA(cudaGetLastError());
  act_backward_kernel<<<flat_grid((size_t)B * kFcIn), 256, 0, st>>>(g_a4, L.u4, (size_t)B * kFcIn, kSqrt2, g_a4);
  NFI_CUDA(cudaGetLastError());
  const float g4w = conv_gain(kCat, 3);
  if (gw_b4 || gb_b4) {
    b4_conv_dw_kernel<<<blocks((size_t)kC4 * kCat * 9, 256), 256, 0, st>>>(g_a4, xs, g4w, B, gw_b4, gb_b4);
    NFI_CUDA(cudaGetLastError());
  }
  b4_conv_dx_kernel<<<dim3(blocks(kCat, 256), (unsigned)B), 256, 0, st>>>(g_a4, P.b4_conv_w, g4w, g_xs);
  NFI_CUDA(cudaGetLastError());
  mbstd_backward_kernel<<<blocks((size_t)B / kGroup * kFcIn, 256), 256, 0, st>>>(g_xs, L.x4, B, V.gA);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// What the weight gradients pair the reverse walk's g with, per block and at fromrgb: the saved
// forward's activations and image, or in the HVP their tangents.
struct Acts {
  const Pair *x, *ph, *d;
  const float* img;
};

// The blocks' reverse walk, last to first, and fromrgb's, over `copies` stacked copies of the B
// images, from g of the last block's output in V.gA.  Term k of a weight gradient pairs acts[k] with
// gradient copy copies - 1 - k: the first order's one term is g (x) a, the HVP's two are g-dot (x) a
// and g (x) a-dot.  A bias pairs with a constant, so its gradient, like the image's, takes the last
// copy alone.  Below block 0 only what is asked for runs.
static int reverse_walk(const nfi_disc_params& P, const Layout& L, const Reverse& V, int copies, const Acts* acts,
                        float* grad_img, const nfi_disc_grads& G, cudaStream_t st) {
  const int B = P.batch, R = P.resolution, nc = P.img_channels, nb = n_blocks(R);
  float* gy = V.gA;  // the gradient of the current block's output
  for (int i = nb - 1; i >= 0; --i) {
    const BlockShape s = shape(R, i);
    const int M = B * s.h * s.h, Mr = B * s.r * s.r;
    const size_t mo = (size_t)M * s.Co, mr = (size_t)Mr * s.C, mf = (size_t)B * (s.r + 1) * (s.r + 1) * s.C;
    float* gx = gy == V.gA ? V.gB : V.gA;
    const bool below = i > 0 || grad_img || G.fromrgb_w || G.fromrgb_b;
    for (int c = 0; c < copies; ++c) {
      out_backward_kernel<<<blocks(M, kRows), 256, 0, st>>>(gy + c * mo, L.u1[i], M, s.Co, V.gy.hi + c * mo,
                                                            V.gy.lo + c * mo, V.gu.hi + c * mo, V.gu.lo + c * mo,
                                                            V.bpart);
      NFI_CUDA(cudaGetLastError());
    }
    if (int rc = synth::bias_reduce(V.bpart, blocks(M, kRows), s.Co, G.conv1_b[i], st)) return rc;
    if (int rc = synth::wgrad_terms(G.conv1_w[i], copies, [&](int k) {
          return synth::wgrad_down3x3(B, s.h, s.C, s.Co, acts[k].ph[i], shifted(V.gu, (copies - 1 - k) * mo), V.part,
                                      V.wtmp, st);
        }, s.Co, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kCiCoTap, V.wtmp, st))
      return rc;
    if (int rc = synth::wgrad_terms(G.skip_w[i], copies, [&](int k) {
          return synth::wgrad1x1(B, s.h, s.Co, s.C, shifted(V.gy, (copies - 1 - k) * mo), acts[k].d[i], V.part,
                                 V.wtmp, st);
        }, s.Co, s.C, 1, s.C, conv_gain(s.C, 1) * kSkipGain, synth::kCoCiTap, V.wtmp, st))
      return rc;
    if (below || G.conv0_w[i] || G.conv0_b[i]) {
      if (int rc = synth::prep_weights(P.conv1_w[i], s.Co, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCiCo,
                                       V.t1, st))
        return rc;
      if (int rc = synth::conv_up3x3(copies * B, s.h, s.Co, s.C, V.gu, V.t1, V.gf, st)) return rc;
      for (int c = 0; c < copies; ++c) {
        fir_up_act_kernel<<<blocks(Mr, kRows), 256, 0, st>>>(V.gf + c * mf, L.a[i].hi, B, s.r, s.C,
                                                             V.g0.hi + c * mr, V.g0.lo + c * mr, V.bpart);
        NFI_CUDA(cudaGetLastError());
      }
      if (int rc = synth::bias_reduce(V.bpart, blocks(Mr, kRows), s.C, G.conv0_b[i], st)) return rc;
      if (int rc = synth::wgrad_terms(G.conv0_w[i], copies, [&](int k) {
            return synth::wgrad3x3(B, s.r, s.r, s.C, s.C, s.C, shifted(V.g0, (copies - 1 - k) * mr), acts[k].x[i],
                                   V.part, V.wtmp, st);
          }, s.C, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kCoCiTap, V.wtmp, st))
        return rc;
    }
    if (!below) break;
    if (int rc = synth::prep_weights(P.conv0_w[i], s.C, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCiCo, V.t0, st))
      return rc;
    if (int rc = synth::conv3x3_adjoint(copies * B, s.r, s.r, s.C, s.C, V.g0, V.t0, gx, st)) return rc;
    if (int rc = synth::prep_weights(P.skip_w[i], s.Co, s.C, 1, s.C, conv_gain(s.C, 1) * kSkipGain, synth::kTapCiCo,
                                     V.ts, st))
      return rc;
    if (int rc = synth::conv1x1(copies * B, s.h, s.Co, s.C, V.gy, V.ts, V.gd, st)) return rc;
    fir_down_adjoint_kernel<<<flat_grid(copies * mr), 256, 0, st>>>(V.gd, copies * B, s.r, s.C, gx);
    NFI_CUDA(cudaGetLastError());
    gy = gx;
  }
  // ---- fromrgb: gy is now the gradient of its output
  const int C = channels(R), RR = R * R, n = (int)blocks((size_t)B * RR, kRows);
  const float grgb = 1.f / sqrtf((float)nc);
  const size_t m0 = (size_t)B * RR * C;
  for (int k = 0; k < copies; ++k) {
    float* g_b = k == 0 ? G.fromrgb_b : nullptr;
    if (!G.fromrgb_w && !g_b) continue;
    fromrgb_backward_kernel<<<n, 256, 0, st>>>(gy + (copies - 1 - k) * m0, L.x[0].hi, acts[k].img, B, nc, RR, C,
                                               V.bpart);
    NFI_CUDA(cudaGetLastError());
    fromrgb_reduce_kernel<<<blocks((size_t)C * (1 + nc), 256), 256, 0, st>>>(V.bpart, n, C, nc, grgb, G.fromrgb_w,
                                                                             g_b);
    NFI_CUDA(cudaGetLastError());
  }
  if (grad_img) {
    fromrgb_gimg_kernel<<<flat_grid((size_t)B * RR * 32), 256, 0, st>>>(gy + (copies - 1) * m0, L.x[0].hi,
                                                                        P.fromrgb_w, grgb, B, nc, RR, C, grad_img);
    NFI_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace

int forward(const nfi_disc_params& P, cudaStream_t st) {
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const int B = P.batch, R = P.resolution, nc = P.img_channels, nb = n_blocks(R);
  const int N = P.cmap_dim ? P.cmap_dim : 1;
  {
    const int C = channels(R);
    fromrgb_kernel<<<flat_grid((size_t)B * R * R * C), 256, 0, st>>>(
        P.img, B, nc, R * R, C, P.fromrgb_w, 1.f / sqrtf((float)nc), P.fromrgb_b, L.x[0].hi, L.x[0].lo);
    NFI_CUDA(cudaGetLastError());
  }
  for (int i = 0; i < nb; ++i) {
    const BlockShape s = shape(R, i);
    const size_t hh = (size_t)B * s.h * s.h;
    if (int rc = synth::prep_weights(P.conv0_w[i], s.C, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCoCi, L.w0, st))
      return rc;
    if (int rc = synth::prep_weights(P.conv1_w[i], s.Co, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCoCi, L.w1, st))
      return rc;
    if (int rc = synth::prep_weights(P.skip_w[i], s.Co, s.C, 1, s.C, conv_gain(s.C, 1) * kSkipGain, synth::kTapCoCi,
                                     L.ws, st))
      return rc;
    if (int rc = synth::conv3x3_act(B, s.r, s.r, s.C, s.C, L.x[i], L.w0, P.conv0_b[i], kSqrt2, kSlope, L.a[i], st))
      return rc;
    fir_phases_kernel<<<flat_grid((size_t)4 * B * (s.h + 1) * (s.h + 1) * s.C), 256, 0, st>>>(
        L.a[i].hi, L.a[i].lo, B, s.r, s.C, L.ph[i].hi, L.ph[i].lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv_down3x3(B, s.h, s.C, s.Co, L.ph[i], L.w1, L.raw1, st)) return rc;
    fir_down_kernel<<<flat_grid(hh * s.C), 256, 0, st>>>(L.x[i].hi, L.x[i].lo, B, s.r, s.C, L.d[i].hi, L.d[i].lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv1x1(B, s.h, s.C, s.Co, L.d[i], L.ws, L.raws, st)) return rc;
    const bool last = i == nb - 1;
    block_out_kernel<<<flat_grid(hh * s.Co), 256, 0, st>>>(L.raw1, L.raws, P.conv1_b[i], hh * s.Co, s.Co, L.u1[i],
                                                           last ? nullptr : L.x[i + 1].hi,
                                                           last ? nullptr : L.x[i + 1].lo, last ? L.x4 : nullptr);
    NFI_CUDA(cudaGetLastError());
  }
  mbstd_kernel<<<B / kGroup, 256, 0, st>>>(L.x4, B, L.xs, L.sd);
  NFI_CUDA(cudaGetLastError());
  w4_kernel<<<flat_grid((size_t)kC4 * kCat * 9), 256, 0, st>>>(P.b4_conv_w, conv_gain(kCat, 3), L.wt4);
  NFI_CUDA(cudaGetLastError());
  b4_conv_kernel<<<dim3((unsigned)B, kC4 / 64), 256, 0, st>>>(L.xs, L.wt4, P.b4_conv_b, L.u4, L.a4);
  NFI_CUDA(cudaGetLastError());
  const unsigned bgrid = blocks(B, kLinImg);
  linear_kernel<<<dim3(kC4, bgrid), 256, 0, st>>>(L.a4, P.fc_w, 1.f / sqrtf((float)kFcIn), P.fc_b, B, kFcIn, kC4,
                                                  1, L.uf, L.hf);
  NFI_CUDA(cudaGetLastError());
  linear_kernel<<<dim3((unsigned)N, bgrid), 256, 0, st>>>(L.hf, P.out_w, 1.f / sqrtf((float)kC4), P.out_b, B, kC4,
                                                          N, 0, nullptr, L.out);
  NFI_CUDA(cudaGetLastError());
  logits_kernel<<<blocks(B, 128), 128, 0, st>>>(L.out, P.cmap, B, P.cmap_dim, P.logits);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int backward(const nfi_disc_params& P, const float* g_logits, float* grad_img, float* grad_cmap,
             const nfi_disc_grads& G, cudaStream_t st) {
  if (!P.save) return fail("discriminator backward: needs the workspace of a forward with save = 1");
  if (!g_logits) return fail("discriminator backward: g_logits must be set");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  if (int rc = epilogue_backward(P, L, L.rev, g_logits, L.hf, L.a4, L.xs, G.out_w, G.fc_w, G.b4_conv_w, G.out_b,
                                 G.fc_b, G.b4_conv_b, grad_cmap, st))
    return rc;
  const Acts saved = {L.x, L.ph, L.d, P.img};
  return reverse_walk(P, L, L.rev, 1, &saved, grad_img, G, st);
}

int saved_preactivation(const nfi_disc_params& P, int block, int which, float* out, cudaStream_t st) {
  const int nb = n_blocks(P.resolution);
  const bool ok = P.save && out != nullptr && block >= 0 && block <= nb && which >= 0 &&
                  ((block < nb && which <= 2 && (which > 0 || block == 0)) || (block == nb && which <= 1));
  if (!ok)
    return fail("discriminator saved_preactivation: needs a saved forward, out, and a block in "
                "0..%d with which in 1..2 (0..2 for block 0, 0..1 for the 4x4 epilogue)", nb);
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const size_t B = P.batch;
  size_t n;
  const __nv_bfloat16 *hi = nullptr, *lo = nullptr;
  const float* u = nullptr;
  if (block == nb) {
    n = which == 0 ? B * kFcIn : B * kC4;
    u = which == 0 ? L.u4 : L.uf;
  } else {
    const BlockShape s = shape(P.resolution, block);
    if (which == 2) {
      n = B * s.h * s.h * s.Co;
      u = L.u1[block];
    } else {
      n = B * s.r * s.r * s.C;
      const Pair p = which == 0 ? L.x[0] : L.a[block];
      hi = p.hi;
      lo = p.lo;
    }
  }
  unpack_kernel<<<flat_grid(n), 256, 0, st>>>(hi, lo, u, n, out);
  NFI_CUDA(cudaGetLastError());
  return 0;
}


// ================================================================ R1: the double backward
// (C ABI: include/nfi_disc_r1.h).  With L = sum_b g_logits[b] logits[b] and a tangent t of the
// image, the pass returns the gradients of Phi = <t, dL/dimg>: the tangent of every first-order
// gradient along img + eps t.  Three properties of the network keep it small:
//   1. every layer but the minibatch std is piecewise linear in the image; on the saved forward's
//      leaky-ReLU branches lrelu'' = 0, so a layer's tangent is its linear map times lrelu';
//   2. above the minibatch std the first-order cotangents (g_out = g_logits cmap / sqrt N, g_hf,
//      g_uf, g_a4, g_u4, g_xs and the std channel's g_sd) do not depend on the image: their
//      tangents are zero.  So the epilogue's weight terms are g (x) a-dot only (xs-dot for the
//      conv, a4-dot for fc, hf-dot for out), its three biases get exactly zero, and
//      dPhi/dcmap = g_logits out-dot / sqrt N;
//   3. the minibatch std is the one second-order kernel: with v = mean_k (x_k - mu)^2 over a group
//      of 4 and s = sqrt(v + 1e-8) its backward is G_j / (16 * 512) (x_k - mu) / (4 s); its tangent
//      along x4-dot seeds the blocks' reverse walk, where g-dot runs through the same linear maps
//      as g.
// Kernels:
//   tangent forward from t, on the saved branches: fromrgb_tangent_kernel; conv0 RAW
//   (nfi::synth::conv3x3, zero bias) then act_tangent_kernel; fir_phases_kernel and conv1
//   (conv_down3x3); fir_down_kernel and the skip (conv1x1); block_out_tangent_kernel;
//   mbstd_tangent_kernel; b4_conv_kernel / linear_kernel with a zero bias, then
//   act_backward_kernel for the branches; logits_kernel (J_img t, the g_logits gradient).
//   dPhi/dcmap: logits_backward_kernel on out-dot.
//   reverse walk: the first-order backward's, with two copies.  epilogue_backward (g, its weight
//   terms against the tangents) ends in mbstd_backward_kernel (g), and mbstd_hvp_kernel (g-dot)
//   fills the second half of the stacked [g; g-dot] buffer of 2B images.  reverse_walk runs the
//   data GEMMs and fir_down_adjoint_kernel once over the 2B images, the pointwise passes per copy
//   with the g-dot copy's bias partials, and each weight's gradient g-dot (x) a + g (x) a-dot as two
//   wgrad_* launches into one buffer and one finish.
// Reads a save = 1 workspace only; everything it writes but the caller's outputs is the scratch.
namespace {

// x-dot[b,p,c] = sqrt2 lrelu'(x) sum_ci (w[c,ci] g) t[b,ci,p] -> pair [B,R,R,C]
__global__ void __launch_bounds__(256)
fromrgb_tangent_kernel(const float* __restrict__ t, int B, int nc, int RR, int C, const float* __restrict__ w,
                       float g, const __nv_bfloat16* __restrict__ xhi, __nv_bfloat16* __restrict__ hi,
                       __nv_bfloat16* __restrict__ lo) {
  const size_t total = (size_t)B * RR * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t q = i / C;
    const int p = (int)(q % RR);
    const size_t b = q / RR;
    float s = 0.f;
    for (int ci = 0; ci < nc; ++ci) s += (__ldg(w + c * nc + ci) * g) * __ldg(t + (b * nc + ci) * RR + p);
    split_bf16(s * kSqrt2 * branch(xhi, i), hi[i], lo[i]);
  }
}

// a-dot = gain lrelu'(a) raw -> pair
__global__ void __launch_bounds__(256)
act_tangent_kernel(const float* __restrict__ raw, const __nv_bfloat16* __restrict__ ahi, size_t n, float gain,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    split_bf16(__ldg(raw + i) * gain * branch(ahi, i), hi[i], lo[i]);
}

// y-dot = lrelu'(u1) u1-dot + skip-dot -> pair and / or fp32
__global__ void __launch_bounds__(256)
block_out_tangent_kernel(const float* __restrict__ raw1, const float* __restrict__ skip,
                         const float* __restrict__ u1, size_t n, __nv_bfloat16* __restrict__ hi,
                         __nv_bfloat16* __restrict__ lo, float* __restrict__ y_out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float y = __ldg(skip + i) + __ldg(raw1 + i) * lrelu_grad(__ldg(u1 + i), kSlope);
    if (hi != nullptr) split_bf16(y, hi[i], lo[i]);
    if (y_out != nullptr) y_out[i] = y;
  }
}

// The minibatch std's tangent: sd-dot[j] = mean over (p, c) of sum_k (x_k - m)(x-dot_k - m-dot) / (4 s),
// in mbstd_kernel's order; xs-dot [B,16,513] = x-dot and sd-dot.  One block per group.
__global__ void __launch_bounds__(256)
mbstd_tangent_kernel(const float* __restrict__ x, const float* __restrict__ dx, int B, float* __restrict__ dxs) {
  __shared__ float part[256];
  const int G = B / kGroup, j = blockIdx.x;
  float s = 0.f;
  for (int e = threadIdx.x; e < 16 * kC4; e += 256) {
    const Group q = group(x, dx, G, j, e);
    s += q.dvar / ((float)kGroup * q.s);
    for (int k = 0; k < kGroup; ++k) dxs[((size_t)(k * G + j) * 16 + e / kC4) * kCat + e % kC4] = q.dv[k];
  }
  part[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < kGroup * 16) {
    const int k = threadIdx.x / 16, p = threadIdx.x % 16;
    dxs[((size_t)(k * G + j) * 16 + p) * kCat + kC4] = part[0] / (float)(16 * kC4);
  }
}

// The tangent of mbstd_backward_kernel's g_x along x-dot (g_xs does not move): with G_j as there,
// g-dot_x = G_j / (16 * 512 * 4) ((x-dot_k - m-dot) / s - (x_k - m) s-dot / s^2),
// s-dot = sum_k (x_k - m)(x-dot_k - m-dot) / (4 s).  Thread per (group, e).
__global__ void mbstd_hvp_kernel(const float* __restrict__ gxs, const float* __restrict__ x,
                                 const float* __restrict__ dx, int B, float* __restrict__ dgx) {
  const int G = B / kGroup;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * 16 * kC4) return;
  const int e = (int)(i % (16 * kC4)), j = (int)(i / (16 * kC4));
  const float gs = std_grad_sum(gxs, G, j);
  const Group q = group(x, dx, G, j, e);
  const float ds = q.dvar / ((float)kGroup * q.s);
  const float c = gs / (float)(16 * kC4) / (float)kGroup;
  for (int k = 0; k < kGroup; ++k)
    dgx[(size_t)(k * G + j) * 16 * kC4 + e] = c * ((q.dv[k] - q.dm) / q.s - (q.v[k] - q.m) * ds / (q.s * q.s));
}

__global__ void accumulate_kernel(const float* __restrict__ src, int n, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}

// The scratch: the tangent forward's activations per block, its weights, and the reverse walk's
// buffers for the stacked [g; g-dot].
struct HvpLayout {
  Pair dx[kMaxBlocks], da[kMaxBlocks], dph[kMaxBlocks], dd[kMaxBlocks];  // as Layout's x, a, ph, d
  Pair w0, w1, ws;
  float* raw0;                   // [B,r,r,C] conv0's raw tangent
  float* raw1;
  float* raws;
  float* zero;                   // [512] zero bias
  float *dx4, *dxs, *du4, *junk, *da4, *dhf, *dout, *jt;
  Reverse rev;
};

void hvp_layout(const nfi_disc_params& P, Bump& b, HvpLayout& L) {
  memset(&L, 0, sizeof(L));
  const Sizes z = sizes(P);
  const size_t B = P.batch, N = P.cmap_dim ? P.cmap_dim : 1;
  for (int i = 0; i < n_blocks(P.resolution); ++i) {
    const BlockShape s = shape(P.resolution, i);
    const size_t rr = (size_t)s.r * s.r, hh = (size_t)s.h * s.h;
    L.dx[i] = b.pair(B * rr * s.C);
    L.da[i] = b.pair(B * rr * s.C);
    L.dph[i] = b.pair(4 * B * (s.h + 1) * (s.h + 1) * s.C);
    L.dd[i] = b.pair(B * hh * s.C);
  }
  L.w0 = b.pair(z.bigw);
  L.w1 = b.pair(z.bigw);
  L.ws = b.pair(z.bigw / 9);
  L.raw0 = b.take(z.big);
  L.raw1 = b.take(z.bigo);
  L.raws = b.take(z.bigo);
  L.zero = b.take(kC4);
  L.dx4 = b.take(B * kFcIn);
  L.dxs = b.take(B * 16 * kCat);
  L.du4 = b.take(B * kFcIn);
  L.junk = b.take(B * kFcIn);
  L.da4 = b.take(B * kFcIn);
  L.dhf = b.take(B * kC4);
  L.dout = b.take(B * N);
  L.jt = b.take(B);
  reverse_layout(P, z, 2, b, L.rev);
}

}  // namespace

size_t hvp_scratch_bytes(const nfi_disc_params& P) {
  if (check(P)) return 0;
  Bump b{nullptr, 0, 0};
  HvpLayout H;
  hvp_layout(P, b, H);
  return b.off + 1024;
}

int backward_hvp(const nfi_disc_params& P, const nfi_disc_hvp& V, const nfi_disc_grads& G, cudaStream_t st) {
  if (P.save != 1) return fail("discriminator HVP: needs the workspace of a forward with save = 1");
  if (!V.g_logits || !V.t_img || !V.scratch) return fail("discriminator HVP: g_logits, t_img and scratch must be set");
  Layout L;
  if (const int rc = setup(P, L)) return rc;
  const size_t need = hvp_scratch_bytes(P);
  if (V.scratch_bytes < need)
    return fail("discriminator HVP: scratch too small (%zu < %zu bytes)", V.scratch_bytes, need);
  HvpLayout H;
  Bump sb = aligned_bump(V.scratch, V.scratch_bytes);
  hvp_layout(P, sb, H);
  const int B = P.batch, R = P.resolution, nc = P.img_channels, nb = n_blocks(R);
  const int N = P.cmap_dim ? P.cmap_dim : 1;
  const int C = channels(R), RR = R * R;
  const float grgb = 1.f / sqrtf((float)nc);
  NFI_CUDA(cudaMemsetAsync(H.zero, 0, kC4 * sizeof(float), st));
  // ---- the tangent forward along t, on the saved branches
  fromrgb_tangent_kernel<<<flat_grid((size_t)B * RR * C), 256, 0, st>>>(V.t_img, B, nc, RR, C, P.fromrgb_w, grgb,
                                                                       L.x[0].hi, H.dx[0].hi, H.dx[0].lo);
  NFI_CUDA(cudaGetLastError());
  for (int i = 0; i < nb; ++i) {
    const BlockShape s = shape(R, i);
    const size_t rr = (size_t)B * s.r * s.r, hh = (size_t)B * s.h * s.h;
    if (int rc = synth::prep_weights(P.conv0_w[i], s.C, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCoCi, H.w0, st))
      return rc;
    if (int rc = synth::prep_weights(P.conv1_w[i], s.Co, s.C, 9, 9 * s.C, conv_gain(s.C, 3), synth::kTapCoCi, H.w1, st))
      return rc;
    if (int rc = synth::prep_weights(P.skip_w[i], s.Co, s.C, 1, s.C, conv_gain(s.C, 1) * kSkipGain, synth::kTapCoCi,
                                     H.ws, st))
      return rc;
    if (int rc = synth::conv3x3(B, s.r, s.r, s.C, s.C, H.dx[i], H.w0, H.zero, H.raw0, Pair{nullptr, nullptr}, st))
      return rc;
    act_tangent_kernel<<<flat_grid(rr * s.C), 256, 0, st>>>(H.raw0, L.a[i].hi, rr * s.C, kSqrt2, H.da[i].hi,
                                                            H.da[i].lo);
    NFI_CUDA(cudaGetLastError());
    fir_phases_kernel<<<flat_grid((size_t)4 * B * (s.h + 1) * (s.h + 1) * s.C), 256, 0, st>>>(
        H.da[i].hi, H.da[i].lo, B, s.r, s.C, H.dph[i].hi, H.dph[i].lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv_down3x3(B, s.h, s.C, s.Co, H.dph[i], H.w1, H.raw1, st)) return rc;
    fir_down_kernel<<<flat_grid(hh * s.C), 256, 0, st>>>(H.dx[i].hi, H.dx[i].lo, B, s.r, s.C, H.dd[i].hi,
                                                         H.dd[i].lo);
    NFI_CUDA(cudaGetLastError());
    if (int rc = synth::conv1x1(B, s.h, s.C, s.Co, H.dd[i], H.ws, H.raws, st)) return rc;
    const bool last = i == nb - 1;
    block_out_tangent_kernel<<<flat_grid(hh * s.Co), 256, 0, st>>>(
        H.raw1, H.raws, L.u1[i], hh * s.Co, last ? nullptr : H.dx[i + 1].hi, last ? nullptr : H.dx[i + 1].lo,
        last ? H.dx4 : nullptr);
    NFI_CUDA(cudaGetLastError());
  }
  mbstd_tangent_kernel<<<B / kGroup, 256, 0, st>>>(L.x4, H.dx4, B, H.dxs);
  NFI_CUDA(cudaGetLastError());
  b4_conv_kernel<<<dim3((unsigned)B, kC4 / 64), 256, 0, st>>>(H.dxs, L.wt4, H.zero, H.du4, H.junk);
  NFI_CUDA(cudaGetLastError());
  act_backward_kernel<<<flat_grid((size_t)B * kFcIn), 256, 0, st>>>(H.du4, L.u4, (size_t)B * kFcIn, 1.f, H.da4);
  NFI_CUDA(cudaGetLastError());
  const unsigned bgrid = blocks(B, kLinImg);
  const float g_out_w = 1.f / sqrtf((float)kC4), g_fc_w = 1.f / sqrtf((float)kFcIn);
  linear_kernel<<<dim3(kC4, bgrid), 256, 0, st>>>(H.da4, P.fc_w, g_fc_w, H.zero, B, kFcIn, kC4, 0, nullptr, H.dhf);
  NFI_CUDA(cudaGetLastError());
  act_backward_kernel<<<flat_grid((size_t)B * kC4), 256, 0, st>>>(H.dhf, L.uf, (size_t)B * kC4, kSqrt2, H.dhf);
  NFI_CUDA(cudaGetLastError());
  linear_kernel<<<dim3((unsigned)N, bgrid), 256, 0, st>>>(H.dhf, P.out_w, g_out_w, H.zero, B, kC4, N, 0, nullptr,
                                                          H.dout);
  NFI_CUDA(cudaGetLastError());
  if (V.grad_g_logits) {
    logits_kernel<<<blocks(B, 128), 128, 0, st>>>(H.dout, P.cmap, B, P.cmap_dim, H.jt);
    NFI_CUDA(cudaGetLastError());
    accumulate_kernel<<<blocks(B, 128), 128, 0, st>>>(H.jt, B, V.grad_g_logits);
    NFI_CUDA(cudaGetLastError());
  }
  if (V.grad_cmap && P.cmap_dim) {  // g_logits out-dot / sqrt N (g_out's write here is discarded)
    logits_backward_kernel<<<blocks((size_t)B * N, 256), 256, 0, st>>>(V.g_logits, H.dout, P.cmap, B, P.cmap_dim,
                                                                       H.junk, V.grad_cmap);
    NFI_CUDA(cudaGetLastError());
  }
  // ---- the reverse walk: the epilogue's g as in the first-order backward (its g-dot is zero, property
  // 2), the minibatch std's g-dot after it, then the blocks over the stacked [g; g-dot]
  if (int rc = epilogue_backward(P, L, H.rev, V.g_logits, H.dhf, H.da4, H.dxs, G.out_w, G.fc_w, G.b4_conv_w,
                                 nullptr, nullptr, nullptr, nullptr, st))
    return rc;
  mbstd_hvp_kernel<<<blocks((size_t)B / kGroup * kFcIn, 256), 256, 0, st>>>(H.rev.g4[3], L.x4, H.dx4, B,
                                                                            H.rev.gA + (size_t)B * kFcIn);
  NFI_CUDA(cudaGetLastError());
  const Acts acts[2] = {{L.x, L.ph, L.d, P.img}, {H.dx, H.dph, H.dd, V.t_img}};
  return reverse_walk(P, L, H.rev, 2, acts, V.grad_img, G, st);
}

}  // namespace disc
}  // namespace nfi

using nfi::fail;

extern "C" {

size_t nfi_disc_workspace_bytes(const nfi_disc_params* params) {
  if (params == nullptr) return 0;
  return nfi::disc::workspace_bytes(*params);
}

int nfi_disc_forward(const nfi_disc_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::disc::forward(*params, (cudaStream_t)stream);
}

int nfi_disc_backward(const nfi_disc_params* params, const float* g_logits, float* grad_img, float* grad_cmap,
                      const nfi_disc_grads* grads, void* stream) {
  if (params == nullptr || grads == nullptr) return fail("params / grads is NULL");
  return nfi::disc::backward(*params, g_logits, grad_img, grad_cmap, *grads, (cudaStream_t)stream);
}

int nfi_disc_saved_preactivation(const nfi_disc_params* params, int32_t block, int32_t which, float* out,
                                 void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::disc::saved_preactivation(*params, block, which, out, (cudaStream_t)stream);
}

size_t nfi_disc_r1_scratch_bytes(const nfi_disc_params* params) {
  if (params == nullptr) return 0;
  return nfi::disc::hvp_scratch_bytes(*params);
}

int nfi_disc_backward_hvp(const nfi_disc_params* params, const nfi_disc_hvp* hvp, const nfi_disc_grads* grads,
                          void* stream) {
  if (params == nullptr || hvp == nullptr || grads == nullptr) return fail("params / hvp / grads is NULL");
  return nfi::disc::backward_hvp(*params, *hvp, *grads, (cudaStream_t)stream);
}

}  // extern "C"
