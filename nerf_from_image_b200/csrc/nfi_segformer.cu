// The bootstrap encoder's SegFormer-B5 backbone on sm_90a (C ABI: include/nfi_segformer.h),
// restating the reference's models/segformer.py:175-275.  Tokens are channel-last rows [M = B N, C];
// every token GEMM runs on the M rows as [Mp / 256, 16, 16, C] (Mp: M rounded up to 256, the extra
// rows zero in every pair a GEMM reads).
//
// Forward, stage i at r = H / 2^(i+2) (M = B r^2 tokens, C = 64 / 128 / 320 / 512):
//   pe1_kernel / phases_kernel + conv_down3x3   patch embed (7x7 s4 in fp32 / 3x3 s2 on the conv kernel)
//   ln_kernel        s = x + scale (y + bias), LN(s) -> the next GEMM's pair (and the stream, stats)
//   conv1x1          q, kv, proj, fc1, fc2 (RAW, weights by synth::prep_weights)
//   s2d_kernel       sr x sr space-to-depth of norm1's pair, then conv1x1 with K = sr^2 C, ln_kernel
//   attn_kernel      softmax(q k^T / 8) v per (image, head, 32-query chunk), keys in shared memory
//   dw_gelu_kernel   depthwise 3x3 of (fc1 + bias), + bias, exact GELU -> pair (pre-GELU kept)
//   head             linear_c_i and linear_fuse's slice i at stage i's resolution (conv1x1),
//                    upsample_sum_kernel (bilinear to r_0, summed, + fuse bias), linear_pred,
//                    synth::transpose -> features [B,out,r0,r0]
// Backward (every sum over positions in a fixed order; no atomics): the same walk reversed.
//   act_kernel           a gradient times the drop-path scale -> pair, per-chunk column sums
//   wgrad_tc_kernel      every GEMM's weight gradient (wgrad1x1, wgrad_down3x3)
//   conv_tc_kernel RAW   data gradients (conv1x1 with transposed weights, conv_up3x3)
//   ln_backward_kernel   LN input gradient (+ the residual's), per-chunk sums for the affine
//   attn_backward_kernel P recomputed; dS = P (dP - rowsum(dO O)); dQ; per-chunk dK, dV that
//                        attn_reduce_kernel adds in chunk order
//   dw_backward_kernel / dw_adjoint_kernel   GELU' and the depthwise conv's three gradients
//   upsample_adjoint_kernel                  the head's bilinear upsample, transposed
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include "nfi_pair.cuh"
#include "nfi_segformer.h"
#include "nfi_synth_launch.h"

namespace nfi {
namespace segformer {
namespace {

constexpr int kStages = NFI_SEGFORMER_STAGES;
constexpr int kMaxDepth = NFI_SEGFORMER_MAX_DEPTH;
constexpr int kDec = NFI_SEGFORMER_DECODER;
constexpr int kDims[kStages] = {64, 128, 320, 512};
constexpr int kSr[kStages] = {8, 4, 2, 1};
constexpr int kD = 64;         // head dimension in every stage
constexpr int kLd = kD + 1;    // shared-memory row pitch of the attention tiles
constexpr int kQ = 32;         // queries per attention block
constexpr int kMaxKeys = 64;
constexpr int kRows = 256;     // the GEMM row quantum; positions per pe1_wgrad_kernel chunk
constexpr int kChunk = 64;     // rows per chunk of the column-sum kernels (8 warps, 32 columns a pass)
constexpr int kLnRows = 8;     // rows per ln_backward_kernel chunk (one per warp)
constexpr int kPe1 = 7, kPe1In = 3, kPe1W = kDims[0] * kPe1In * kPe1 * kPe1;  // 9408 weights
constexpr float kEpsBlock = 1e-6f, kEpsEmbed = 1e-5f;  // block / stage norms; patch embed / attn.norm

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float gelu(float z) { return 0.5f * z * (1.f + erff(z * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_d(float z) {
  return 0.5f * (1.f + erff(z * 0.70710678118654752f)) + z * 0.39894228040143268f * expf(-0.5f * z * z);
}

// ---- patch embed 1: 7x7, stride 4, pad 3, 3 -> 64 channels, fp32.  y [B,r,r,64] (no bias)
__global__ void __launch_bounds__(256)
pe1_kernel(const float* __restrict__ img, const float* __restrict__ w, int B, int H, int r, float* __restrict__ y) {
  __shared__ float ws[kPe1W];
  for (int i = threadIdx.x; i < kPe1W; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const size_t total = (size_t)B * r * r * kDims[0];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int co = (int)(i & 63);
    const size_t p = i >> 6;
    const int ox = (int)(p % r), oy = (int)((p / r) % r);
    const size_t b = p / ((size_t)r * r);
    float s = 0.f;
    for (int ci = 0; ci < kPe1In; ++ci)
      for (int ky = 0; ky < kPe1; ++ky) {
        const int iy = 4 * oy + ky - 3;
        if (iy < 0 || iy >= H) continue;
        for (int kx = 0; kx < kPe1; ++kx) {
          const int ix = 4 * ox + kx - 3;
          if (ix < 0 || ix >= H) continue;
          s += ws[((co * kPe1In + ci) * kPe1 + ky) * kPe1 + kx] * __ldg(img + ((b * kPe1In + ci) * H + iy) * H + ix);
        }
      }
    y[i] = s;
  }
}

// its weight gradient over a chunk of kRows positions: partial[chunk][co][ci][ky][kx]
__global__ void __launch_bounds__(256)
pe1_wgrad_kernel(const float* __restrict__ gy, const float* __restrict__ img, int B, int H, int r,
                 float* __restrict__ partial) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kPe1W) return;
  const int co = j & 63, q = j >> 6, kx = q % kPe1, ky = (q / kPe1) % kPe1, ci = q / (kPe1 * kPe1);
  const size_t M = (size_t)B * r * r, p0 = (size_t)blockIdx.y * kRows;
  const size_t p1 = p0 + kRows < M ? p0 + kRows : M;
  float s = 0.f;
  for (size_t p = p0; p < p1; ++p) {
    const int ox = (int)(p % r), oy = (int)((p / r) % r);
    const size_t b = p / ((size_t)r * r);
    const int iy = 4 * oy + ky - 3, ix = 4 * ox + kx - 3;
    if (iy < 0 || iy >= H || ix < 0 || ix >= H) continue;
    s += __ldg(gy + p * 64 + co) * __ldg(img + ((b * kPe1In + ci) * H + iy) * H + ix);
  }
  partial[(size_t)blockIdx.y * kPe1W + co * (kPe1W / 64) + q] = s;
}

// The zero-padded [B,2h+1,2h+1,C] input of a 3x3 stride-2 pad-1 conv of x [B,2h,2h,C] as its four
// parity phases [4B,h+1,h+1,C] (phase (py,px) at image offset (2py+px) B), the conv_down3x3 layout
__global__ void __launch_bounds__(256)
phases_kernel(const float* __restrict__ x, int B, int h, int C, __nv_bfloat16* __restrict__ hi,
              __nv_bfloat16* __restrict__ lo) {
  const int h1 = h + 1, r = 2 * h;
  const size_t total = (size_t)4 * B * h1 * h1 * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t q = i / C;
    const int n = (int)(q % h1);
    q /= h1;
    const int m = (int)(q % h1);
    q /= h1;
    const int b = (int)(q % B), ph = (int)(q / B);
    const int y = 2 * m + (ph >> 1) - 1, xx = 2 * n + (ph & 1) - 1;
    const float v = (y >= 0 && y < r && xx >= 0 && xx < r) ? __ldg(x + (((size_t)b * r + y) * r + xx) * C + c) : 0.f;
    split_bf16(v, hi[i], lo[i]);
  }
}

// out [B,2h,2h,C] += gf [B,2h+1,2h+1,C] at (y+1, x+1): the data gradient through the padding
__global__ void __launch_bounds__(256)
crop_add_kernel(const float* __restrict__ gf, int B, int h, int C, float* __restrict__ out) {
  const int r = 2 * h, r1 = r + 1;
  const size_t total = (size_t)B * r * r * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t p = i / C;
    const int x = (int)(p % r), y = (int)((p / r) % r);
    const size_t b = p / ((size_t)r * r);
    out[i] += __ldg(gf + ((b * r1 + y + 1) * r1 + x + 1) * C + c);
  }
}

// ---- LayerNorm.  s = x + scale[b] (y + bias) (each term optional), LN(s) with the affine
struct LnFwd {
  int M, rows, C, per_img;  // valid rows; rows of the pair (zero beyond M); channels; rows per image
  const float* x;
  const float* y;
  const float* bias;
  const float* scale;
  float* s_out;             // s (may be y)
  const float* w;
  const float* b;
  float eps;
  float* out;               // LN(s) fp32
  Pair pair;                // LN(s) pair
  float2* stats;            // (mean, 1 / sqrt(var + eps))
};

// one warp per row
__global__ void __launch_bounds__(256) ln_kernel(const LnFwd a) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, n = a.C >> 5;
  if (r >= a.rows) return;
  const size_t base = (size_t)r * a.C;
  if (r >= a.M) {
    for (int c = lane; c < a.C; c += 32) a.pair.hi[base + c] = a.pair.lo[base + c] = __float2bfloat16_rn(0.f);
    return;
  }
  const float sc = a.scale ? __ldg(a.scale + r / a.per_img) : 1.f;
  float v[16];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (k >= n) break;
    const int c = lane + 32 * k;
    float s = a.x ? a.x[base + c] : 0.f;
    if (a.y) s += sc * (a.y[base + c] + (a.bias ? __ldg(a.bias + c) : 0.f));
    v[k] = s;
    sum += s;
  }
  const float mean = warp_sum(sum) / (float)a.C;
  float var = 0.f;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (k >= n) break;
    var += (v[k] - mean) * (v[k] - mean);
  }
  const float rstd = 1.f / sqrtf(warp_sum(var) / (float)a.C + a.eps);
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (k >= n) break;
    const int c = lane + 32 * k;
    if (a.s_out) a.s_out[base + c] = v[k];
    const float t = (v[k] - mean) * rstd * __ldg(a.w + c) + __ldg(a.b + c);
    if (a.out) a.out[base + c] = t;
    if (a.pair.hi) split_bf16(t, a.pair.hi[base + c], a.pair.lo[base + c]);
  }
  if (lane == 0) a.stats[r] = make_float2(mean, rstd);
}

struct LnBwd {
  int M, C;
  const float* s;        // the saved LN input
  const float2* stats;
  const float* w;
  const float* g;        // the output gradient is g + g2 (g2 optional)
  const float* g2;
  const float* g_res;    // added to the input gradient (optional; may be out)
  float* out;            // the input gradient (may be g or g_res)
  float* partial;        // [chunks][2C]: sums of g xhat, then of g, over the chunk's rows
};

// a chunk of kLnRows rows per block, one warp per row; the affine sums per warp, then in warp order
__global__ void __launch_bounds__(256) ln_backward_kernel(const LnBwd a) {
  __shared__ float red[8][2 * 512];
  const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31, n = a.C >> 5;
  float aw[16], ab[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) aw[k] = ab[k] = 0.f;
  for (int rr = wp; rr < kLnRows; rr += 8) {
    const int r = blockIdx.x * kLnRows + rr;
    if (r >= a.M) break;
    const size_t base = (size_t)r * a.C;
    const float2 st = a.stats[r];
    float gx[16], xh[16];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (k >= n) break;
      const int c = lane + 32 * k;
      const float g = a.g[base + c] + (a.g2 ? a.g2[base + c] : 0.f);
      xh[k] = (a.s[base + c] - st.x) * st.y;
      gx[k] = g * __ldg(a.w + c);
      aw[k] += g * xh[k];
      ab[k] += g;
      s1 += gx[k];
      s2 += gx[k] * xh[k];
    }
    s1 = warp_sum(s1) / (float)a.C;
    s2 = warp_sum(s2) / (float)a.C;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (k >= n) break;
      const int c = lane + 32 * k;
      const float res = a.g_res ? a.g_res[base + c] : 0.f;
      a.out[base + c] = res + st.y * (gx[k] - s1 - xh[k] * s2);
    }
  }
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (k >= n) break;
    red[wp][lane + 32 * k] = aw[k];
    red[wp][a.C + lane + 32 * k] = ab[k];
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * a.C; j += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][j];
    a.partial[(size_t)blockIdx.x * 2 * a.C + j] = s;
  }
}

// sum_k partial[k stride + j] over the chunks: a block per 32 columns, warp w summing chunks w,
// w + 8, ... in order, then the eight warps' sums in warp order
__device__ __forceinline__ float chunk_sum(const float* __restrict__ partial, int chunks, int stride, int n, int j) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  float s = 0.f;
  if (j < n)
    for (int k = wp; k < chunks; k += 8) s += partial[(size_t)k * stride + j];
  red[wp][lane] = s;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < 8; ++w) t += red[w][lane];
  return t;
}

// out[j] += the chunks' sum of column j
__global__ void __launch_bounds__(256)
reduce_kernel(const float* __restrict__ partial, int chunks, int stride, int n, float* __restrict__ out) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const float t = chunk_sum(partial, chunks, stride, n, j);
  if (threadIdx.x < 32 && j < n) out[j] += t;
}

// v = (g + bias) scale[b] over the first M of `rows` rows (0 beyond) -> pair, and per-chunk column
// sums of v.  One block per (kChunk rows, 32 adjacent columns): a warp's lanes take the columns,
// its rows every eighth, and the eight warps' sums are added in warp order.
struct Act {
  int M, rows, C, per_img;
  const float* g;
  const float* bias;
  const float* scale;
  Pair out;
  float* partial;
};
__global__ void __launch_bounds__(256) act_kernel(const Act a) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * kChunk, r1 = min(a.rows, r0 + kChunk), c = blockIdx.y * 32 + lane;
  const float bc = a.bias ? __ldg(a.bias + c) : 0.f;
  float s = 0.f;
  for (int r = r0 + wp; r < r1; r += 8) {
    const size_t o = (size_t)r * a.C + c;
    float v = 0.f;
    if (r < a.M) {
      v = a.g[o] + bc;
      if (a.scale) v *= __ldg(a.scale + r / a.per_img);
      s += v;
    }
    if (a.out.hi) split_bf16(v, a.out.hi[o], a.out.lo[o]);
  }
  if (a.partial) {
    red[wp][lane] = s;
    __syncthreads();
    if (wp == 0) {
      float t = 0.f;
      for (int w = 0; w < 8; ++w) t += red[w][lane];
      a.partial[(size_t)blockIdx.x * a.C + c] = t;
    }
  }
}

// norm1's pair [B,r,r,C] -> [B,r/sr,r/sr,sr^2 C] (rows beyond Mr of `rows` zero), column
// (ky sr + kx) C + c; the values are copied, so they are the pair q reads
__global__ void __launch_bounds__(256)
s2d_kernel(Pair in, int B, int r, int sr, int C, int rows, Pair out) {
  const int rr = r / sr, K = sr * sr * C;
  const size_t Mr = (size_t)B * rr * rr, total = (size_t)rows * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / K;
    if (row >= Mr) {
      out.hi[i] = out.lo[i] = __float2bfloat16_rn(0.f);
      continue;
    }
    const int k = (int)(i % K), t = k / C, c = k % C, J = (int)(row % rr), I = (int)((row / rr) % rr);
    const size_t b = row / ((size_t)rr * rr);
    const size_t src = ((b * r + I * sr + t / sr) * r + J * sr + t % sr) * C + c;
    out.hi[i] = in.hi[src];
    out.lo[i] = in.lo[src];
  }
}

// its adjoint on fp32: g [Mr, sr^2 C] -> out [B,r,r,C] (every position is one column of one row)
__global__ void __launch_bounds__(256)
d2s_kernel(const float* __restrict__ g, int B, int r, int sr, int C, float* __restrict__ out) {
  const int rr = r / sr, K = sr * sr * C;
  const size_t total = (size_t)B * rr * rr * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / K;
    const int k = (int)(i % K), t = k / C, c = k % C, J = (int)(row % rr), I = (int)((row / rr) % rr);
    const size_t b = row / ((size_t)rr * rr);
    out[((b * r + I * sr + t / sr) * r + J * sr + t % sr) * C + c] = g[i];
  }
}

// ---- attention, per (32-query chunk, head, image).  q [M,C] and kv [Mr,2C] are GEMM outputs
// without their biases; the 1/8 scale is folded into q (a power of two: exact)
struct AttnTiles {
  float *K, *V, *Q, *P;
};
__device__ __forceinline__ AttnTiles attn_load(float* sm, const float* q, const float* bq, const float* kv,
                                               const float* bkv, int N, int Nk, int C, int nq) {
  AttnTiles t;
  t.K = sm;
  t.V = t.K + kMaxKeys * kLd;
  t.Q = t.V + kMaxKeys * kLd;
  t.P = t.Q + kQ * kLd;
  const int h = blockIdx.y, b = blockIdx.z, i0 = blockIdx.x * kQ;
  for (int e = threadIdx.x; e < Nk * kD; e += blockDim.x) {
    const int j = e >> 6, d = e & 63;
    const size_t row = ((size_t)b * Nk + j) * 2 * C + h * kD + d;
    t.K[j * kLd + d] = kv[row] + __ldg(bkv + h * kD + d);
    t.V[j * kLd + d] = kv[row + C] + __ldg(bkv + C + h * kD + d);
  }
  for (int e = threadIdx.x; e < nq * kD; e += blockDim.x) {
    const int i = e >> 6, d = e & 63;
    t.Q[i * kLd + d] = (q[((size_t)b * N + i0 + i) * C + h * kD + d] + __ldg(bq + h * kD + d)) * 0.125f;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nq * Nk; e += blockDim.x) {
    const int i = e / Nk, j = e % Nk;
    float s = 0.f;
    for (int d = 0; d < kD; ++d) s += t.Q[i * kLd + d] * t.K[j * kLd + d];
    t.P[i * kLd + j] = s;
  }
  __syncthreads();
  const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = wp; i < nq; i += blockDim.x >> 5) {
    const float s0 = lane < Nk ? t.P[i * kLd + lane] : -INFINITY;
    const float s1 = lane + 32 < Nk ? t.P[i * kLd + lane + 32] : -INFINITY;
    const float m = warp_max(fmaxf(s0, s1));
    const float e0 = lane < Nk ? expf(s0 - m) : 0.f, e1 = lane + 32 < Nk ? expf(s1 - m) : 0.f;
    const float sum = warp_sum(e0 + e1);
    if (lane < Nk) t.P[i * kLd + lane] = e0 / sum;
    if (lane + 32 < Nk) t.P[i * kLd + lane + 32] = e1 / sum;
  }
  __syncthreads();
  return t;
}
constexpr int kAttnSmem = (2 * kMaxKeys + 2 * kQ) * kLd * 4;
constexpr int kAttnBwdSmem = (2 * kMaxKeys + 4 * kQ) * kLd * 4 + kQ * 4;

__global__ void __launch_bounds__(256)
attn_kernel(const float* __restrict__ q, const float* __restrict__ bq, const float* __restrict__ kv,
            const float* __restrict__ bkv, int N, int Nk, int C, float* __restrict__ o, Pair op) {
  extern __shared__ float sm[];
  const int i0 = blockIdx.x * kQ, nq = min(kQ, N - i0), h = blockIdx.y, b = blockIdx.z;
  const AttnTiles t = attn_load(sm, q, bq, kv, bkv, N, Nk, C, nq);
  for (int e = threadIdx.x; e < nq * kD; e += blockDim.x) {
    const int i = e >> 6, d = e & 63;
    float s = 0.f;
    for (int j = 0; j < Nk; ++j) s += t.P[i * kLd + j] * t.V[j * kLd + d];
    const size_t oo = ((size_t)b * N + i0 + i) * C + h * kD + d;
    o[oo] = s;
    split_bf16(s, op.hi[oo], op.lo[oo]);
  }
}

// dq [M,C] (written), and this chunk's dK, dV [Nk][64] to part[((b heads + h) chunks + chunk)][2]
__global__ void __launch_bounds__(256)
attn_backward_kernel(const float* __restrict__ q, const float* __restrict__ bq, const float* __restrict__ kv,
                     const float* __restrict__ bkv, const float* __restrict__ o, const float* __restrict__ go,
                     int N, int Nk, int C, float* __restrict__ gq, float* __restrict__ part) {
  extern __shared__ float sm[];
  const int i0 = blockIdx.x * kQ, nq = min(kQ, N - i0), h = blockIdx.y, b = blockIdx.z;
  const AttnTiles t = attn_load(sm, q, bq, kv, bkv, N, Nk, C, nq);
  float* dO = t.P + kQ * kLd;
  float* dS = dO + kQ * kLd;
  float* Dr = dS + kQ * kLd;
  for (int e = threadIdx.x; e < nq * kD; e += blockDim.x) {
    const int i = e >> 6, d = e & 63;
    dO[i * kLd + d] = go[((size_t)b * N + i0 + i) * C + h * kD + d];
  }
  __syncthreads();
  // rowsum(dO o) in the order of dP's sums below: with one key o is v exactly, so dS is exactly 0
  for (int i = threadIdx.x; i < nq; i += blockDim.x) {
    const float* oi = o + ((size_t)b * N + i0 + i) * C + h * kD;
    float s = 0.f;
    for (int d = 0; d < kD; ++d) s += dO[i * kLd + d] * oi[d];
    Dr[i] = s;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nq * Nk; e += blockDim.x) {
    const int i = e / Nk, j = e % Nk;
    float s = 0.f;
    for (int d = 0; d < kD; ++d) s += dO[i * kLd + d] * t.V[j * kLd + d];
    dS[i * kLd + j] = t.P[i * kLd + j] * (s - Dr[i]);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nq * kD; e += blockDim.x) {
    const int i = e >> 6, d = e & 63;
    float s = 0.f;
    for (int j = 0; j < Nk; ++j) s += dS[i * kLd + j] * t.K[j * kLd + d];
    gq[((size_t)b * N + i0 + i) * C + h * kD + d] = 0.125f * s;
  }
  float* pk = part + (((size_t)b * gridDim.y + h) * gridDim.x + blockIdx.x) * 2 * Nk * kD;
  for (int e = threadIdx.x; e < Nk * kD; e += blockDim.x) {
    const int j = e >> 6, d = e & 63;
    float sk = 0.f, sv = 0.f;
    for (int i = 0; i < nq; ++i) {
      sk += dS[i * kLd + j] * t.Q[i * kLd + d];
      sv += t.P[i * kLd + j] * dO[i * kLd + d];
    }
    pk[e] = sk;
    pk[Nk * kD + e] = sv;
  }
}

// gkv [Mr,2C] = the chunks' dK, dV summed in chunk order
__global__ void __launch_bounds__(256)
attn_reduce_kernel(const float* __restrict__ part, int B, int heads, int chunks, int Nk, int C, float* __restrict__ gkv) {
  const size_t total = (size_t)B * Nk * 2 * C;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / (2 * C);
    const int col = (int)(e % (2 * C)), tk = col / C, hc = col % C, h = hc / kD, d = hc % kD;
    const int j = (int)(row % Nk);
    const size_t b = row / Nk;
    float s = 0.f;
    for (int k = 0; k < chunks; ++k)
      s += part[((((b * heads + h) * chunks + k) * 2 + tk) * Nk + j) * kD + d];
    gkv[e] = s;
  }
}

// ---- MLP's depthwise 3x3 (pad 1) of hb = fc1 + b1, + bias, exact GELU -> pair (rows >= M zero)
__global__ void __launch_bounds__(256)
dw_gelu_kernel(const float* __restrict__ h, const float* __restrict__ b1, const float* __restrict__ w,
               const float* __restrict__ bw, int B, int r, int C, int rows, float* __restrict__ z, Pair out) {
  const size_t M = (size_t)B * r * r, total = (size_t)rows * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i / C;
    if (p >= M) {
      out.hi[i] = out.lo[i] = __float2bfloat16_rn(0.f);
      continue;
    }
    const int c = (int)(i % C), x = (int)(p % r), y = (int)((p / r) % r);
    const size_t b = p / ((size_t)r * r);
    const float bc = __ldg(b1 + c);
    float s = 0.f;
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y + ky - 1;
      if (yy < 0 || yy >= r) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = x + kx - 1;
        if (xx < 0 || xx >= r) continue;
        s += __ldg(w + c * 9 + ky * 3 + kx) * (h[((b * r + yy) * r + xx) * C + c] + bc);
      }
    }
    s += __ldg(bw + c);
    z[i] = s;
    split_bf16(gelu(s), out.hi[i], out.lo[i]);
  }
}

// g (the GELU output's gradient) -> gz = g gelu'(z) in place; per-chunk sums of gz hb(tap) for the
// weight and of gz for the bias: partial[chunk][10][C].  Threads as in act_kernel.
__global__ void __launch_bounds__(256)
dw_backward_kernel(float* __restrict__ g, const float* __restrict__ z, const float* __restrict__ h,
                   const float* __restrict__ b1, int B, int r, int C, float* __restrict__ partial) {
  __shared__ float red[8][10][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int M = B * r * r, p0 = blockIdx.x * kChunk, p1 = min(M, p0 + kChunk), c = blockIdx.y * 32 + lane;
  float pw[10];
#pragma unroll
  for (int t = 0; t < 10; ++t) pw[t] = 0.f;
  const float bc = __ldg(b1 + c);
  for (int p = p0 + wp; p < p1; p += 8) {
    const size_t o = (size_t)p * C + c;
    const float gz = g[o] * gelu_d(z[o]);
    g[o] = gz;
    pw[9] += gz;
    const int x = p % r, y = (p / r) % r, b = p / (r * r);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy < 0 || yy >= r || xx < 0 || xx >= r) continue;
      pw[t] += gz * (h[(((size_t)b * r + yy) * r + xx) * C + c] + bc);
    }
  }
#pragma unroll
  for (int t = 0; t < 10; ++t) red[wp][t][lane] = pw[t];
  __syncthreads();
  for (int t = wp; t < 10; t += 8) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][t][lane];
    partial[((size_t)blockIdx.x * 10 + t) * C + c] = s;
  }
}

// the data gradient of the depthwise conv: ghb[p] = sum_t w[t] gz[p - (t - centre)] -> pair (rows
// >= M of `rows` zero), per-chunk sums for b1.  Threads as in act_kernel.
__global__ void __launch_bounds__(256)
dw_adjoint_kernel(const float* __restrict__ gz, const float* __restrict__ w, int B, int r, int C, int rows,
                  Pair out, float* __restrict__ partial) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int M = B * r * r, p0 = blockIdx.x * kChunk, p1 = min(rows, p0 + kChunk), c = blockIdx.y * 32 + lane;
  float wc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wc[t] = __ldg(w + c * 9 + t);
  float s = 0.f;
  for (int p = p0 + wp; p < p1; p += 8) {
    float v = 0.f;
    if (p < M) {
      const int x = p % r, y = (p / r) % r, b = p / (r * r);
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int yy = y - t / 3 + 1, xx = x - t % 3 + 1;
        if (yy < 0 || yy >= r || xx < 0 || xx >= r) continue;
        v += wc[t] * gz[(((size_t)b * r + yy) * r + xx) * C + c];
      }
      s += v;
    }
    split_bf16(v, out.hi[(size_t)p * C + c], out.lo[(size_t)p * C + c]);
  }
  red[wp][lane] = s;
  __syncthreads();
  if (wp == 0) {
    float t = 0.f;
    for (int w2 = 0; w2 < 8; ++w2) t += red[w2][lane];
    partial[(size_t)blockIdx.x * C + c] = t;
  }
}

// g_w[c][t] += sum_k partial[k][t][c], g_b[c] += sum_k partial[k][9][c] (as reduce_kernel)
__global__ void __launch_bounds__(256)
dw_reduce_kernel(const float* __restrict__ partial, int chunks, int C, float* __restrict__ g_w,
                 float* __restrict__ g_b) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31), t = j / C, c = j % C;
  const float s = chunk_sum(partial, chunks, 10 * C, 10 * C, j);
  if (threadIdx.x >= 32 || j >= 10 * C) return;
  if (t < 9 && g_w) g_w[c * 9 + t] += s;
  if (t == 9 && g_b) g_b[c] += s;
}

// ---- decoder head
struct Head4 {
  const float* d[kStages];  // linear_fuse's slice of stage i at r0 >> i, [B,r_i,r_i,768]
};
// u = d0 + up2(d1) + up4(d2) + up8(d3) + bias -> pair [rows, 768] (rows >= B r0^2 zero)
__global__ void __launch_bounds__(256)
upsample_sum_kernel(const Head4 hd, int B, int r0, const float* __restrict__ bias, int rows, Pair out) {
  const size_t M = (size_t)B * r0 * r0, total = (size_t)rows * kDec;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i / kDec;
    if (p >= M) {
      out.hi[i] = out.lo[i] = __float2bfloat16_rn(0.f);
      continue;
    }
    const int c = (int)(i % kDec), X = (int)(p % r0), Y = (int)((p / r0) % r0);
    const size_t b = p / ((size_t)r0 * r0);
    float acc = hd.d[0][i];
    for (int s = 1; s < kStages; ++s) {
      const int h = r0 >> s;
      const float inv = 1.f / (float)(1 << s);
      int y0, y1, x0, x1;
      float ly0, ly1, lx0, lx1;
      src_index(Y, inv, h, y0, y1, ly0, ly1);
      src_index(X, inv, h, x0, x1, lx0, lx1);
      const float* d = hd.d[s];
      const float v00 = d[((b * h + y0) * h + x0) * kDec + c], v01 = d[((b * h + y0) * h + x1) * kDec + c];
      const float v10 = d[((b * h + y1) * h + x0) * kDec + c], v11 = d[((b * h + y1) * h + x1) * kDec + c];
      acc += ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
    }
    acc += __ldg(bias + c);
    split_bf16(acc, out.hi[i], out.lo[i]);
  }
}

// the adjoint of the upsample by S: g [B,Sh,Sh,768] -> pair [rows, 768] at h (rows >= B h^2 zero)
__global__ void __launch_bounds__(256)
upsample_adjoint_kernel(const float* __restrict__ g, int B, int h, int S, int rows, Pair out) {
  const int Ho = S * h;
  const float inv_s = 1.f / (float)S;
  const size_t M = (size_t)B * h * h, total = (size_t)rows * kDec;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i / kDec;
    float acc = 0.f;
    if (p < M) {
      const int c = (int)(i % kDec), sj = (int)(p % h), si = (int)((p / h) % h);
      const size_t b = p / ((size_t)h * h);
      const int ya = max(0, S * (si - 1)), yb = min(Ho, S * (si + 2));
      const int xa = max(0, S * (sj - 1)), xb = min(Ho, S * (sj + 2));
      for (int Y = ya; Y < yb; ++Y) {
        const float wy = src_weight(Y, si, inv_s, h);
        if (wy == 0.f) continue;
        for (int X = xa; X < xb; ++X) {
          const float wx = src_weight(X, sj, inv_s, h);
          if (wx == 0.f) continue;
          acc += (wy * wx) * __ldg(g + ((b * Ho + Y) * Ho + X) * kDec + c);
        }
      }
    }
    split_bf16(acc, out.hi[i], out.lo[i]);
  }
}

// ---------------------------------------------------------------- host side
static size_t rnd(size_t m) { return (m + kRows - 1) / kRows * kRows; }

struct Shape {
  int r, N, C, heads, sr, rr, Nk, K;  // map side, tokens per image, width, heads, sr, reduced side, keys, sr^2 C
  size_t M, Mp, Mr, Mrp, Mkv;         // tokens, padded; reduced tokens, padded; kv GEMM rows
};
static Shape shape(const nfi_segformer_params& P, int i) {
  Shape s;
  s.r = P.height >> (i + 2);
  s.N = s.r * s.r;
  s.C = kDims[i];
  s.heads = s.C / kD;
  s.sr = kSr[i];
  s.rr = s.r / s.sr;
  s.Nk = s.rr * s.rr;
  s.K = s.sr * s.sr * s.C;
  s.M = (size_t)P.batch * s.N;
  s.Mp = rnd(s.M);
  s.Mr = (size_t)P.batch * s.Nk;
  s.Mrp = rnd(s.Mr);
  s.Mkv = s.sr > 1 ? s.Mrp : s.Mp;
  return s;
}

// Indices into params / grads (named_parameters() order, nfi_segformer.h)
struct Index {
  int pe[kStages], blk[kStages][kMaxDepth], norm[kStages], lc[kStages], fuse, pred, total;
};
static Index index_of(const nfi_segformer_params& P) {
  Index x;
  int n = 0;
  for (int i = 0; i < kStages; ++i, n += 4) x.pe[i] = n;
  for (int i = 0; i < kStages; ++i) {
    for (int k = 0; k < P.depths[i]; ++k, n += kSr[i] > 1 ? 20 : 16) x.blk[i][k] = n;
    x.norm[i] = n;
    n += 2;
  }
  for (int i = kStages - 1; i >= 0; --i, n += 2) x.lc[i] = n;
  x.fuse = n;
  x.pred = n + 2;
  x.total = n + 4;
  return x;
}
// offsets within a block
enum { kN1 = 0, kQw = 2, kKv = 4, kProj = 6, kSrW = 8, kSrN = 10 };
static int blk_off(int sr) { return sr > 1 ? 12 : 8; }  // norm2; then fc1 +2, dwconv +4, fc2 +6

struct Blk {
  float* x;      // the block's input (the residual stream)
  float2* st1;
  Pair a1;       // norm1(x)
  float* q;      // q without bias [Mp,C]
  Pair sd;       // space-to-depth of a1 [Mrp,K]
  float* sr;     // sr conv + bias (attn.norm's input) [Mrp,C]
  float2* str;
  Pair xr;       // attn.norm's output [Mrp,C]
  float* kv;     // [Mkv,2C] without bias
  float* o;      // attention output [M,C]
  Pair op;
  float* x1;     // after the attention branch
  float2* st2;
  Pair a2;       // norm2(x1)
  float* h;      // fc1 without bias [Mp,4C]
  float* z;      // pre-GELU [Mp,4C]
  Pair g;        // GELU [Mp,4C]
};
struct BlkSize {
  size_t m, a, sd, sr, mr, kv, h;
  void max_with(const BlkSize& o) {
    m = m > o.m ? m : o.m; a = a > o.a ? a : o.a; sd = sd > o.sd ? sd : o.sd; sr = sr > o.sr ? sr : o.sr;
    mr = mr > o.mr ? mr : o.mr; kv = kv > o.kv ? kv : o.kv; h = h > o.h ? h : o.h;
  }
};
static BlkSize blk_size(const Shape& s) {
  BlkSize z;
  z.m = s.M * s.C;
  z.a = s.Mp * s.C;
  z.sd = s.sr > 1 ? s.Mrp * s.K : 0;
  z.sr = s.sr > 1 ? s.Mrp * s.C : 0;
  z.mr = s.sr > 1 ? s.Mr : 0;
  z.kv = s.Mkv * 2 * s.C;
  z.h = s.Mp * 4 * s.C;
  return z;
}
static Blk take_blk(Bump& b, const BlkSize& z, size_t M) {
  Blk k;
  memset(&k, 0, sizeof(k));
  k.st1 = reinterpret_cast<float2*>(b.take(2 * M));
  k.a1 = b.pair(z.a);
  k.q = b.take(z.a);
  if (z.sd) {
    k.sd = b.pair(z.sd);
    k.sr = b.take(z.sr);
    k.str = reinterpret_cast<float2*>(b.take(2 * z.mr));
    k.xr = b.pair(z.sr);
  }
  k.kv = b.take(z.kv);
  k.o = b.take(z.m);
  k.op = b.pair(z.a);
  k.x1 = b.take(z.m);
  k.st2 = reinterpret_cast<float2*>(b.take(2 * M));
  k.a2 = b.pair(z.a);
  k.h = b.take(z.h);
  k.z = b.take(z.h);
  k.g = b.pair(z.h);
  return k;
}

struct StageBufs {
  float* pe;      // patch embed conv + bias (its norm's input) [M,C]
  float2* pst;
  Pair ph;        // the phases of the previous stage's features (stages 2-4)
  Blk blk[kMaxDepth];
  float* xs;      // the last block's output (the stage norm's input)
  float2* stn;
  float* feat;    // the stage's features [M,C] fp32
  Pair fp;        // and as a pair [Mp,C]
  Pair cp;        // linear_c_i + bias [Mp,768]
  float* d;       // linear_fuse's slice i [Mp,768]
};
struct Layout {
  StageBufs s[kStages];
  Pair w;         // one GEMM's weight pair
  float* y;       // one GEMM's output
  Pair u;         // linear_fuse's output [M0p,768]
  float* pred;    // linear_pred's output [M0p,out]
  // backward (save only)
  float* gfeat[kStages];
  float *gx, *ga, *gln, *gq, *gkv, *gxr, *gsd, *gext, *gpe, *wtmp, *part, *bpart, *apart;
  Pair gy, gh, gkvp, gsr;
};

static size_t mx(size_t a, size_t b) { return a > b ? a : b; }

static void layout(const nfi_segformer_params& P, Bump& b, Layout& L) {
  memset(&L, 0, sizeof(L));
  const int B = P.batch, out = P.out_features;
  Shape sh[kStages];
  BlkSize all = {0, 0, 0, 0, 0, 0, 0};
  size_t wmax = (size_t)out * kDec, ymax = 0, mc = 0, mpc = 0, mp4c = 0, mpdec = 0, mkv2c = 0, mkvc = 0,
         mrpc = 0, mrpk = 0, mr2c = 0, upmax = 0, tmpmax = (size_t)kDec * kDec, partmax = 0, bpmax = 0, apmax = 0;
  for (int i = 0; i < kStages; ++i) {
    const Shape s = shape(P, i);
    sh[i] = s;
    all.max_with(blk_size(s));
    const size_t C = s.C;
    wmax = mx(wmax, mx(4 * C * C, mx((size_t)s.K * C, (size_t)kDec * C)));
    if (i > 0) {
      wmax = mx(wmax, 9 * C * kDims[i - 1]);
      tmpmax = mx(tmpmax, 9 * C * kDims[i - 1]);
      upmax = mx(upmax, (size_t)B * (2 * s.r + 1) * (2 * s.r + 1) * kDims[i - 1]);
      partmax = mx(partmax, synth::wgrad_down3x3_partial_floats(B, s.r, kDims[i - 1], s.C));
    }
    tmpmax = mx(tmpmax, (size_t)s.K * C);
    ymax = mx(ymax, s.Mp * mx(C, kDec));
    mc = mx(mc, s.M * C);
    mpc = mx(mpc, s.Mp * C);
    mp4c = mx(mp4c, s.Mp * 4 * C);
    mpdec = mx(mpdec, s.Mp * kDec);
    mkv2c = mx(mkv2c, s.Mkv * 2 * C);
    mkvc = mx(mkvc, s.Mkv * C);
    mrpc = mx(mrpc, s.Mrp * C);
    if (s.sr > 1) mrpk = mx(mrpk, s.Mrp * s.K);
    mr2c = mx(mr2c, s.Mr * 2 * C);
    const int B16 = (int)(s.Mp / kRows), Br16 = (int)(s.Mkv / kRows);
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(B16, 16, s.C, s.C));
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(B16, 16, 4 * s.C, s.C));
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(B16, 16, s.C, 4 * s.C));
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(Br16, 16, 2 * s.C, s.C));
    if (s.sr > 1) partmax = mx(partmax, synth::wgrad1x1_partial_floats((int)(s.Mrp / kRows), 16, s.C, s.K));
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(B16, 16, kDec, s.C));
    partmax = mx(partmax, synth::wgrad1x1_partial_floats(B16, 16, kDec, kDec));
    bpmax = mx(bpmax, (size_t)blocks(s.Mp, kChunk) * mx(4 * C, kDec));
    bpmax = mx(bpmax, (size_t)blocks(s.M, kLnRows) * 2 * C);
    bpmax = mx(bpmax, (size_t)blocks(s.M, kChunk) * 10 * 4 * C);
    apmax = mx(apmax, (size_t)B * s.heads * blocks(s.N, kQ) * 2 * s.Nk * kD);
  }
  const Shape& s0 = sh[0];
  partmax = mx(partmax, synth::wgrad1x1_partial_floats((int)(s0.Mp / kRows), 16, out, kDec));
  bpmax = mx(bpmax, (size_t)blocks(s0.Mp, kChunk) * out);
  bpmax = mx(bpmax, (size_t)blocks(s0.M, kRows) * kPe1W);
  upmax = mx(upmax, s0.M * out);

  Blk shared_blk;
  float* shared_x[2] = {nullptr, nullptr};
  if (!P.save) {
    shared_blk = take_blk(b, all, mx(mx(sh[0].M, sh[1].M), mx(sh[2].M, sh[3].M)));
    shared_x[0] = b.take(all.m);
    shared_x[1] = b.take(all.m);
  }
  for (int i = 0; i < kStages; ++i) {
    const Shape& s = sh[i];
    StageBufs& S = L.s[i];
    const int d = P.depths[i];
    S.pe = b.take(s.M * s.C);
    S.pst = reinterpret_cast<float2*>(b.take(2 * s.M));
    if (i > 0) S.ph = b.pair((size_t)4 * B * (s.r + 1) * (s.r + 1) * kDims[i - 1]);
    if (P.save) {
      for (int k = 0; k < d; ++k) {
        S.blk[k] = take_blk(b, blk_size(s), s.M);
        S.blk[k].x = b.take(s.M * s.C);
      }
      S.xs = b.take(s.M * s.C);
    } else {
      for (int k = 0; k < d; ++k) {
        S.blk[k] = shared_blk;
        S.blk[k].x = shared_x[k & 1];
      }
      S.xs = shared_x[d & 1];
    }
    S.stn = reinterpret_cast<float2*>(b.take(2 * s.M));
    S.feat = b.take(s.M * s.C);
    S.fp = b.pair(s.Mp * s.C);
    S.cp = b.pair(s.Mp * kDec);
    S.d = b.take(s.Mp * kDec);
  }
  L.w = b.pair(wmax);
  L.y = b.take(ymax);
  L.u = b.pair(s0.Mp * kDec);
  L.pred = b.take(s0.Mp * out);
  if (P.save) {
    for (int i = 0; i < kStages; ++i) L.gfeat[i] = b.take(sh[i].Mp * sh[i].C);
    L.gx = b.take(mc);
    L.gy = b.pair(mx(mx(mpc, mpdec), s0.Mp * out));
    L.ga = b.take(mx(mp4c, mpdec));
    L.gh = b.pair(mx(mp4c, mpdec));
    L.gln = b.take(mx(mpc, mpdec));
    L.gq = b.take(mc);
    L.gkv = b.take(mr2c);
    L.gkvp = b.pair(mkv2c);
    L.gxr = b.take(mkvc);
    L.gsr = b.pair(mrpc);
    L.gsd = b.take(mrpk);
    L.gext = b.take(mc);
    L.gpe = b.take(upmax);
    L.wtmp = b.take(tmpmax);
    L.part = b.take(partmax);
    L.bpart = b.take(bpmax);
    L.apart = b.take(apmax);
  }
}

static int check(const nfi_segformer_params& P) {
  if (P.batch <= 0 || P.batch > 65535 || P.height != P.width || P.height < 32 || P.height > 256 ||
      P.height % 32 != 0)
    return fail("segformer: B in 1..65535 and a square image with H a multiple of 32 in 32..256 "
                "needed, got B %d, %d x %d", P.batch, P.height, P.width);
  const size_t M0 = (size_t)P.batch * (P.height / 4) * (P.height / 4);
  if (M0 * kDec > (size_t)INT_MAX || M0 * P.out_features > (size_t)INT_MAX)
    return fail("segformer: more than 2^31 head activations (B %d, %d x %d)", P.batch, P.height, P.width);
  for (int i = 0; i < kStages; ++i)
    if (P.depths[i] < 1 || P.depths[i] > kMaxDepth)
      return fail("segformer: depths in 1..%d, got %d in stage %d", kMaxDepth, P.depths[i], i + 1);
  if (P.out_features <= 0 || P.out_features % 64 != 0 || P.out_features > 4096)
    return fail("segformer: out_features must be a multiple of 64 in 64..4096, got %d", P.out_features);
  if (P.save != 0 && P.save != 1) return fail("segformer: save must be 0 or 1, got %d", P.save);
  return 0;
}

}  // namespace

size_t workspace_bytes(const nfi_segformer_params& P) {
  if (check(P)) return 0;
  Bump b{nullptr, 0, 0};
  Layout L;
  layout(P, b, L);
  return b.off + 1024;
}

namespace {

static int setup(const nfi_segformer_params& P, Layout& L, Index& X) {
  if (const int rc = check(P)) return rc;
  if (!P.image || !P.params || !P.features || !P.workspace)
    return fail("segformer: image, params, features and workspace must be set");
  X = index_of(P);
  for (int j = 0; j < X.total; ++j)
    if (!P.params[j]) return fail("segformer: parameter %d of %d is NULL", j, X.total);
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need)
    return fail("segformer: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  Bump b = aligned_bump(P.workspace, P.workspace_bytes);
  layout(P, b, L);
  return 0;
}

// one token GEMM: out [Mp,N] = in [Mp,K] w^T, w the pair [N][K]
static int gemm(size_t Mp, int K, int N, Pair in, Pair w, float* out, cudaStream_t st) {
  return synth::conv1x1((int)(Mp / kRows), 16, K, N, in, w, out, st);
}
// g_w [cout][cin] += g^T x over Mp rows
static int wgrad(size_t Mp, int cout, int cin, Pair g, Pair x, float* part, float* g_w, cudaStream_t st) {
  return synth::wgrad1x1((int)(Mp / kRows), 16, cout, cin, g, x, part, g_w, st);
}
// a linear layer's weight [cout][cin] (row pitch ld) as the pair [cout][cin] of its GEMM, or
// [cin][cout] (transposed) of its data gradient's
static int prep(const float* w, int cout, int cin, int ld, bool transposed, Pair out, cudaStream_t st) {
  return synth::prep_weights(w, cout, cin, 1, ld, 1.f, transposed ? synth::kTapCiCo : synth::kTapCoCi, out, st);
}
static int ln(const LnFwd& a, cudaStream_t st) {
  ln_kernel<<<blocks((size_t)a.rows, 8), 256, 0, st>>>(a);
  NFI_CUDA(cudaGetLastError());
  return 0;
}
static int reduce(const float* partial, int n_chunks, int stride, int n, float* out, cudaStream_t st) {
  if (out == nullptr) return 0;
  reduce_kernel<<<blocks((size_t)n, 32), 256, 0, st>>>(partial, n_chunks, stride, n, out);
  NFI_CUDA(cudaGetLastError());
  return 0;
}
// the LN backward and its affine gradients
static int ln_backward(const LnBwd& a, float* g_w, float* g_b, cudaStream_t st) {
  const unsigned n = blocks((size_t)a.M, kLnRows);
  ln_backward_kernel<<<n, 256, 0, st>>>(a);
  NFI_CUDA(cudaGetLastError());
  if (int rc = reduce(a.partial, (int)n, 2 * a.C, a.C, g_w, st)) return rc;
  return reduce(a.partial + a.C, (int)n, 2 * a.C, a.C, g_b, st);
}
static int act(const Act& a, float* g_b, cudaStream_t st) {
  const unsigned n = blocks((size_t)a.rows, kChunk);
  act_kernel<<<dim3(n, (unsigned)(a.C / 32)), 256, 0, st>>>(a);
  NFI_CUDA(cudaGetLastError());
  return g_b ? reduce(a.partial, (int)n, a.C, a.C, g_b, st) : 0;
}

}  // namespace

int forward(const nfi_segformer_params& P, cudaStream_t st) {
  Layout L;
  Index X;
  if (const int rc = setup(P, L, X)) return rc;
  const float* const* W = P.params;
  const int B = P.batch, H = P.height, out = P.out_features;
  int gk = 0;  // blocks so far (the drop-path scale rows)
  for (int i = 0; i < kStages; ++i) {
    const Shape s = shape(P, i);
    StageBufs& S = L.s[i];
    const int C = s.C, pe = X.pe[i];
    // patch embed -> the stream x0 = blk[0].x
    if (i == 0) {
      pe1_kernel<<<flat_grid(s.M * C), 256, 0, st>>>(P.image, W[pe], B, H, s.r, S.pe);
    } else {
      const int Cp = kDims[i - 1];
      phases_kernel<<<flat_grid((size_t)4 * B * (s.r + 1) * (s.r + 1) * Cp), 256, 0, st>>>(L.s[i - 1].feat, B, s.r,
                                                                                          Cp, S.ph.hi, S.ph.lo);
      NFI_CUDA(cudaGetLastError());
      if (int rc = synth::prep_weights(W[pe], C, Cp, 9, 9 * Cp, 1.f, synth::kTapCoCi, L.w, st))
        return rc;
      if (int rc = synth::conv_down3x3(B, s.r, Cp, C, S.ph, L.w, S.pe, st)) return rc;
    }
    NFI_CUDA(cudaGetLastError());
    LnFwd a;
    memset(&a, 0, sizeof(a));
    a.M = a.rows = (int)s.M; a.C = C; a.per_img = s.N;
    a.y = S.pe; a.bias = W[pe + 1]; a.s_out = S.pe; a.w = W[pe + 2]; a.b = W[pe + 3]; a.eps = kEpsEmbed;
    a.out = S.blk[0].x; a.stats = S.pst;
    if (int rc = ln(a, st)) return rc;
    // norm1 of block 0
    const int nb0 = X.blk[i][0];
    memset(&a, 0, sizeof(a));
    a.M = (int)s.M; a.rows = (int)s.Mp; a.C = C; a.per_img = s.N;
    a.x = S.blk[0].x; a.w = W[nb0 + kN1]; a.b = W[nb0 + kN1 + 1]; a.eps = kEpsBlock;
    a.pair = S.blk[0].a1; a.stats = S.blk[0].st1;
    if (int rc = ln(a, st)) return rc;
    for (int k = 0; k < P.depths[i]; ++k, ++gk) {
      Blk& K = S.blk[k];
      const int nb = X.blk[i][k], o2 = nb + blk_off(s.sr);
      const float* sc_a = P.drop_scales ? P.drop_scales + (size_t)(2 * gk) * B : nullptr;
      const float* sc_m = P.drop_scales ? P.drop_scales + (size_t)(2 * gk + 1) * B : nullptr;
      if (int rc = prep(W[nb + kQw], C, C, C, false, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, C, K.a1, L.w, K.q, st)) return rc;
      Pair kvin = K.a1;
      if (s.sr > 1) {
        s2d_kernel<<<flat_grid(s.Mrp * s.K), 256, 0, st>>>(K.a1, B, s.r, s.sr, C, (int)s.Mrp, K.sd);
        NFI_CUDA(cudaGetLastError());
        if (int rc = synth::prep_weights(W[nb + kSrW], C, C, s.sr * s.sr, s.K, 1.f, synth::kCoTapCi, L.w, st))
          return rc;
        if (int rc = gemm(s.Mrp, s.K, C, K.sd, L.w, K.sr, st)) return rc;
        memset(&a, 0, sizeof(a));
        a.M = (int)s.Mr; a.rows = (int)s.Mrp; a.C = C; a.per_img = s.Nk;
        a.y = K.sr; a.bias = W[nb + kSrW + 1]; a.s_out = K.sr; a.w = W[nb + kSrN]; a.b = W[nb + kSrN + 1];
        a.eps = kEpsEmbed; a.pair = K.xr; a.stats = K.str;
        if (int rc = ln(a, st)) return rc;
        kvin = K.xr;
      }
      if (int rc = prep(W[nb + kKv], 2 * C, C, C, false, L.w, st)) return rc;
      if (int rc = gemm(s.Mkv, C, 2 * C, kvin, L.w, K.kv, st)) return rc;
      NFI_CUDA(cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem));
      attn_kernel<<<dim3(blocks(s.N, kQ), s.heads, B), 256, kAttnSmem, st>>>(K.q, W[nb + kQw + 1], K.kv,
                                                                              W[nb + kKv + 1], s.N, s.Nk, C, K.o, K.op);
      NFI_CUDA(cudaGetLastError());
      if (s.Mp > s.M) {
        const size_t pad = (s.Mp - s.M) * C * sizeof(__nv_bfloat16);
        NFI_CUDA(cudaMemsetAsync(K.op.hi + s.M * C, 0, pad, st));
        NFI_CUDA(cudaMemsetAsync(K.op.lo + s.M * C, 0, pad, st));
      }
      if (int rc = prep(W[nb + kProj], C, C, C, false, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, C, K.op, L.w, L.y, st)) return rc;
      memset(&a, 0, sizeof(a));
      a.M = (int)s.M; a.rows = (int)s.Mp; a.C = C; a.per_img = s.N;
      a.x = K.x; a.y = L.y; a.bias = W[nb + kProj + 1]; a.scale = sc_a; a.s_out = K.x1;
      a.w = W[o2]; a.b = W[o2 + 1]; a.eps = kEpsBlock; a.pair = K.a2; a.stats = K.st2;
      if (int rc = ln(a, st)) return rc;
      if (int rc = prep(W[o2 + 2], 4 * C, C, C, false, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, 4 * C, K.a2, L.w, K.h, st)) return rc;
      dw_gelu_kernel<<<flat_grid(s.Mp * 4 * C), 256, 0, st>>>(K.h, W[o2 + 3], W[o2 + 4], W[o2 + 5], B, s.r, 4 * C,
                                                              (int)s.Mp, K.z, K.g);
      NFI_CUDA(cudaGetLastError());
      if (int rc = prep(W[o2 + 6], C, 4 * C, 4 * C, false, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, 4 * C, C, K.g, L.w, L.y, st)) return rc;
      // the residual, then the next norm: the next block's norm1, or the stage norm
      const bool last = k + 1 == P.depths[i];
      memset(&a, 0, sizeof(a));
      a.M = (int)s.M; a.rows = (int)s.Mp; a.C = C; a.per_img = s.N;
      a.x = K.x1; a.y = L.y; a.bias = W[o2 + 7]; a.scale = sc_m; a.eps = kEpsBlock;
      if (last) {
        a.s_out = S.xs; a.w = W[X.norm[i]]; a.b = W[X.norm[i] + 1]; a.out = S.feat; a.pair = S.fp; a.stats = S.stn;
      } else {
        Blk& N1 = S.blk[k + 1];
        const int nn = X.blk[i][k + 1];
        a.s_out = N1.x; a.w = W[nn + kN1]; a.b = W[nn + kN1 + 1]; a.pair = N1.a1; a.stats = N1.st1;
      }
      if (int rc = ln(a, st)) return rc;
    }
  }
  // decoder head: linear_c_i and linear_fuse's slice at stage i's resolution
  Head4 hd;
  for (int i = 0; i < kStages; ++i) {
    const Shape s = shape(P, i);
    StageBufs& S = L.s[i];
    if (int rc = prep(W[X.lc[i]], kDec, s.C, s.C, false, L.w, st)) return rc;
    if (int rc = gemm(s.Mp, s.C, kDec, S.fp, L.w, L.y, st)) return rc;
    Act c;
    memset(&c, 0, sizeof(c));
    c.M = (int)s.M; c.rows = (int)s.Mp; c.C = kDec; c.per_img = s.N; c.g = L.y; c.bias = W[X.lc[i] + 1]; c.out = S.cp;
    if (int rc = act(c, nullptr, st)) return rc;
    if (int rc = prep(W[X.fuse] + (kStages - 1 - i) * kDec, kDec, kDec, kStages * kDec, false, L.w, st))
      return rc;
    if (int rc = gemm(s.Mp, kDec, kDec, S.cp, L.w, S.d, st)) return rc;
    hd.d[i] = S.d;
  }
  const Shape s0 = shape(P, 0);
  upsample_sum_kernel<<<flat_grid(s0.Mp * kDec), 256, 0, st>>>(hd, B, s0.r, W[X.fuse + 1], (int)s0.Mp, L.u);
  NFI_CUDA(cudaGetLastError());
  if (int rc = prep(W[X.pred], out, kDec, kDec, false, L.w, st)) return rc;
  if (int rc = gemm(s0.Mp, kDec, out, L.u, L.w, L.pred, st)) return rc;
  return synth::transpose(L.pred, B, s0.N, out, W[X.pred + 1], 0, P.features, st);
}

int backward(const nfi_segformer_params& P, const float* g_features, float* const* G, cudaStream_t st) {
  if (!P.save) return fail("segformer backward: needs the workspace of a forward with save = 1");
  if (!g_features || !G) return fail("segformer backward: g_features and grads must be set");
  Layout L;
  Index X;
  if (const int rc = setup(P, L, X)) return rc;
  const float* const* W = P.params;
  const int B = P.batch, H = P.height, out = P.out_features;
  const Shape s0 = shape(P, 0);
  // ---- head
  if (int rc = synth::transpose(g_features, B, out, s0.N, nullptr, 0, L.gpe, st)) return rc;
  Act c;
  memset(&c, 0, sizeof(c));
  c.M = (int)s0.M; c.rows = (int)s0.Mp; c.C = out; c.per_img = s0.N; c.g = L.gpe; c.out = L.gy; c.partial = L.bpart;
  if (int rc = act(c, G[X.pred + 1], st)) return rc;
  if (int rc = wgrad(s0.Mp, out, kDec, L.gy, L.u, L.part, G[X.pred], st)) return rc;
  if (int rc = prep(W[X.pred], out, kDec, kDec, true, L.w, st)) return rc;
  if (int rc = gemm(s0.Mp, out, kDec, L.gy, L.w, L.ga, st)) return rc;
  memset(&c, 0, sizeof(c));
  c.M = (int)s0.M; c.rows = (int)s0.Mp; c.C = kDec; c.per_img = s0.N; c.g = L.ga; c.partial = L.bpart;
  if (int rc = act(c, G[X.fuse + 1], st)) return rc;
  for (int i = 0; i < kStages; ++i) {
    const Shape s = shape(P, i);
    const StageBufs& S = L.s[i];
    if (i == 0) {
      memset(&c, 0, sizeof(c));
      c.M = (int)s.M; c.rows = (int)s.Mp; c.C = kDec; c.per_img = s.N; c.g = L.ga; c.out = L.gh;
      if (int rc = act(c, nullptr, st)) return rc;
    } else {
      upsample_adjoint_kernel<<<flat_grid(s.Mp * kDec), 256, 0, st>>>(L.ga, B, s.r, 1 << i, (int)s.Mp, L.gh);
      NFI_CUDA(cudaGetLastError());
    }
    const float* wf = W[X.fuse] + (kStages - 1 - i) * kDec;
    float* gf = G[X.fuse] ? G[X.fuse] + (kStages - 1 - i) * kDec : nullptr;
    if (int rc = synth::wgrad_terms(gf, 1, [&](int) {
          return wgrad(s.Mp, kDec, kDec, L.gh, S.cp, L.part, L.wtmp, st);
        }, kDec, kDec, 1, kStages * kDec, 1.f, synth::kCoCiTap, L.wtmp, st))
      return rc;
    if (int rc = prep(wf, kDec, kDec, kStages * kDec, true, L.w, st)) return rc;
    if (int rc = gemm(s.Mp, kDec, kDec, L.gh, L.w, L.gln, st)) return rc;
    memset(&c, 0, sizeof(c));
    c.M = (int)s.M; c.rows = (int)s.Mp; c.C = kDec; c.per_img = s.N; c.g = L.gln; c.out = L.gy; c.partial = L.bpart;
    if (int rc = act(c, G[X.lc[i] + 1], st)) return rc;
    if (int rc = wgrad(s.Mp, kDec, s.C, L.gy, S.fp, L.part, G[X.lc[i]], st)) return rc;
    if (int rc = prep(W[X.lc[i]], kDec, s.C, s.C, true, L.w, st)) return rc;
    if (int rc = gemm(s.Mp, kDec, s.C, L.gy, L.w, L.gfeat[i], st)) return rc;
  }
  // ---- stages, last to first
  int gk = 0;
  for (int i = 0; i < kStages; ++i) gk += P.depths[i];
  for (int i = kStages - 1; i >= 0; --i) {
    const Shape s = shape(P, i);
    const StageBufs& S = L.s[i];
    const int C = s.C;
    LnBwd n;
    memset(&n, 0, sizeof(n));
    n.M = (int)s.M; n.C = C; n.s = S.xs; n.stats = S.stn; n.w = W[X.norm[i]]; n.g = L.gfeat[i]; n.out = L.gx;
    n.partial = L.bpart;
    if (int rc = ln_backward(n, G[X.norm[i]], G[X.norm[i] + 1], st)) return rc;
    for (int k = P.depths[i] - 1; k >= 0; --k) {
      --gk;
      const Blk& K = S.blk[k];
      const int nb = X.blk[i][k], o2 = nb + blk_off(s.sr);
      const float* sc_a = P.drop_scales ? P.drop_scales + (size_t)(2 * gk) * B : nullptr;
      const float* sc_m = P.drop_scales ? P.drop_scales + (size_t)(2 * gk + 1) * B : nullptr;
      // MLP branch
      memset(&c, 0, sizeof(c));
      c.M = (int)s.M; c.rows = (int)s.Mp; c.C = C; c.per_img = s.N; c.g = L.gx; c.scale = sc_m; c.out = L.gy;
      c.partial = L.bpart;
      if (int rc = act(c, G[o2 + 7], st)) return rc;
      if (int rc = wgrad(s.Mp, C, 4 * C, L.gy, K.g, L.part, G[o2 + 6], st)) return rc;
      if (int rc = prep(W[o2 + 6], C, 4 * C, 4 * C, true, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, 4 * C, L.gy, L.w, L.ga, st)) return rc;
      const unsigned ndw = blocks(s.M, kChunk);
      dw_backward_kernel<<<dim3(ndw, (unsigned)(4 * C / 32)), 256, 0, st>>>(L.ga, K.z, K.h, W[o2 + 3], B, s.r, 4 * C, L.bpart);
      NFI_CUDA(cudaGetLastError());
      if (G[o2 + 4] || G[o2 + 5]) {
        dw_reduce_kernel<<<blocks((size_t)40 * C, 32), 256, 0, st>>>(L.bpart, (int)ndw, 4 * C, G[o2 + 4], G[o2 + 5]);
        NFI_CUDA(cudaGetLastError());
      }
      const unsigned nadj = blocks(s.Mp, kChunk);
      dw_adjoint_kernel<<<dim3(nadj, (unsigned)(4 * C / 32)), 256, 0, st>>>(L.ga, W[o2 + 4], B, s.r, 4 * C, (int)s.Mp, L.gh, L.bpart);
      NFI_CUDA(cudaGetLastError());
      if (int rc = reduce(L.bpart, (int)nadj, 4 * C, 4 * C, G[o2 + 3], st)) return rc;
      if (int rc = wgrad(s.Mp, 4 * C, C, L.gh, K.a2, L.part, G[o2 + 2], st)) return rc;
      if (int rc = prep(W[o2 + 2], 4 * C, C, C, true, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, 4 * C, C, L.gh, L.w, L.gln, st)) return rc;
      memset(&n, 0, sizeof(n));
      n.M = (int)s.M; n.C = C; n.s = K.x1; n.stats = K.st2; n.w = W[o2]; n.g = L.gln; n.g_res = L.gx; n.out = L.gx;
      n.partial = L.bpart;
      if (int rc = ln_backward(n, G[o2], G[o2 + 1], st)) return rc;
      // attention branch
      memset(&c, 0, sizeof(c));
      c.M = (int)s.M; c.rows = (int)s.Mp; c.C = C; c.per_img = s.N; c.g = L.gx; c.scale = sc_a; c.out = L.gy;
      c.partial = L.bpart;
      if (int rc = act(c, G[nb + kProj + 1], st)) return rc;
      if (int rc = wgrad(s.Mp, C, C, L.gy, K.op, L.part, G[nb + kProj], st)) return rc;
      if (int rc = prep(W[nb + kProj], C, C, C, true, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, C, L.gy, L.w, L.gln, st)) return rc;
      const unsigned nq = blocks(s.N, kQ);
      NFI_CUDA(
  cudaFuncSetAttribute(attn_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnBwdSmem));
      attn_backward_kernel<<<dim3(nq, s.heads, B), 256, kAttnBwdSmem, st>>>(
          K.q, W[nb + kQw + 1], K.kv, W[nb + kKv + 1], K.o, L.gln, s.N, s.Nk, C, L.gq, L.apart);
      NFI_CUDA(cudaGetLastError());
      attn_reduce_kernel<<<flat_grid(s.Mr * 2 * C), 256, 0, st>>>(L.apart, B, s.heads, (int)nq, s.Nk, C, L.gkv);
      NFI_CUDA(cudaGetLastError());
      memset(&c, 0, sizeof(c));
      c.M = (int)s.M; c.rows = (int)s.Mp; c.C = C; c.per_img = s.N; c.g = L.gq; c.out = L.gy; c.partial = L.bpart;
      if (int rc = act(c, G[nb + kQw + 1], st)) return rc;
      if (int rc = wgrad(s.Mp, C, C, L.gy, K.a1, L.part, G[nb + kQw], st)) return rc;
      memset(&c, 0, sizeof(c));
      c.M = (int)s.Mr; c.rows = (int)s.Mkv; c.C = 2 * C; c.per_img = s.Nk; c.g = L.gkv; c.out = L.gkvp;
      c.partial = L.bpart;
      if (int rc = act(c, G[nb + kKv + 1], st)) return rc;
      const Pair kvin = s.sr > 1 ? K.xr : K.a1;
      if (int rc = wgrad(s.Mkv, 2 * C, C, L.gkvp, kvin, L.part, G[nb + kKv], st)) return rc;
      if (int rc = prep(W[nb + kQw], C, C, C, true, L.w, st)) return rc;
      if (int rc = gemm(s.Mp, C, C, L.gy, L.w, L.gln, st)) return rc;
      if (int rc = prep(W[nb + kKv], 2 * C, C, C, true, L.w, st)) return rc;
      if (int rc = gemm(s.Mkv, 2 * C, C, L.gkvp, L.w, L.gxr, st)) return rc;
      const float* g2 = L.gxr;
      if (s.sr > 1) {
        memset(&n, 0, sizeof(n));
        n.M = (int)s.Mr; n.C = C; n.s = K.sr; n.stats = K.str; n.w = W[nb + kSrN]; n.g = L.gxr; n.out = L.gxr;
        n.partial = L.bpart;
        if (int rc = ln_backward(n, G[nb + kSrN], G[nb + kSrN + 1], st)) return rc;
        memset(&c, 0, sizeof(c));
        c.M = (int)s.Mr; c.rows = (int)s.Mrp; c.C = C; c.per_img = s.Nk; c.g = L.gxr; c.out = L.gsr;
        c.partial = L.bpart;
        if (int rc = act(c, G[nb + kSrW + 1], st)) return rc;
        if (int rc = synth::wgrad_terms(G[nb + kSrW], 1, [&](int) {
              return wgrad(s.Mrp, C, s.K, L.gsr, K.sd, L.part, L.wtmp, st);
            }, C, C, s.sr * s.sr, s.K, 1.f, synth::kCoTapCi, L.wtmp, st))
          return rc;
        if (int rc = synth::prep_weights(W[nb + kSrW], C, C, s.sr * s.sr, s.K, 1.f, synth::kTapCiCo, L.w, st))
          return rc;
        if (int rc = gemm(s.Mrp, C, s.K, L.gsr, L.w, L.gsd, st)) return rc;
        d2s_kernel<<<flat_grid(s.Mr * s.K), 256, 0, st>>>(L.gsd, B, s.r, s.sr, C, L.gext);
        NFI_CUDA(cudaGetLastError());
        g2 = L.gext;
      }
      memset(&n, 0, sizeof(n));
      n.M = (int)s.M; n.C = C; n.s = K.x; n.stats = K.st1; n.w = W[nb + kN1]; n.g = L.gln; n.g2 = g2;
      n.g_res = L.gx; n.out = L.gx; n.partial = L.bpart;
      if (int rc = ln_backward(n, G[nb + kN1], G[nb + kN1 + 1], st)) return rc;
    }
    // patch embed: its norm, then the conv
    const int pe = X.pe[i];
    memset(&n, 0, sizeof(n));
    n.M = (int)s.M; n.C = C; n.s = S.pe; n.stats = S.pst; n.w = W[pe + 2]; n.g = L.gx; n.out = L.gx;
    n.partial = L.bpart;
    if (int rc = ln_backward(n, G[pe + 2], G[pe + 3], st)) return rc;
    if (i == 0) {
      memset(&c, 0, sizeof(c));
      c.M = c.rows = (int)s.M; c.C = C; c.per_img = s.N; c.g = L.gx; c.partial = L.bpart;
      if (int rc = act(c, G[pe + 1], st)) return rc;
      if (G[pe]) {
        const unsigned np = blocks(s.M, kRows);
        pe1_wgrad_kernel<<<dim3(blocks(kPe1W, 256), np), 256, 0, st>>>(L.gx, P.image, B, H, s.r, L.bpart);
        NFI_CUDA(cudaGetLastError());
        if (int rc = reduce(L.bpart, (int)np, kPe1W, kPe1W, G[pe], st)) return rc;
      }
    } else {
      const int Cp = kDims[i - 1];
      memset(&c, 0, sizeof(c));
      c.M = c.rows = (int)s.M; c.C = C; c.per_img = s.N; c.g = L.gx; c.out = L.gy; c.partial = L.bpart;
      if (int rc = act(c, G[pe + 1], st)) return rc;
      if (int rc = synth::wgrad_terms(G[pe], 1, [&](int) {
            return synth::wgrad_down3x3(B, s.r, Cp, C, S.ph, L.gy, L.part, L.wtmp, st);
          }, C, Cp, 9, 9 * Cp, 1.f, synth::kCiCoTap, L.wtmp, st))
        return rc;
      if (int rc = synth::prep_weights(W[pe], C, Cp, 9, 9 * Cp, 1.f, synth::kTapCiCo, L.w, st))
        return rc;
      if (int rc = synth::conv_up3x3(B, s.r, C, Cp, L.gy, L.w, L.gpe, st)) return rc;
      crop_add_kernel<<<flat_grid((size_t)B * 4 * s.r * s.r * Cp), 256, 0, st>>>(L.gpe, B, s.r, Cp, L.gfeat[i - 1]);
      NFI_CUDA(cudaGetLastError());
    }
  }
  return 0;
}

}  // namespace segformer
}  // namespace nfi

using nfi::fail;

extern "C" {

size_t nfi_segformer_workspace_bytes(const nfi_segformer_params* params) {
  if (params == nullptr) return 0;
  return nfi::segformer::workspace_bytes(*params);
}

int nfi_segformer_forward(const nfi_segformer_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::segformer::forward(*params, (cudaStream_t)stream);
}

int nfi_segformer_backward(const nfi_segformer_params* params, const float* g_features, float* const* grads,
                           void* stream) {
  if (params == nullptr) return fail("params is NULL");
  return nfi::segformer::backward(*params, g_features, grads, (cudaStream_t)stream);
}

}  // extern "C"
