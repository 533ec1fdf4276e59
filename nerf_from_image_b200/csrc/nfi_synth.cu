// Tri-plane producer on sm_90a: the StyleGAN2 synthesis network of the reference's
// models/stylegan.py:293-490 as TMA-fed wgmma implicit GEMMs (C ABI: include/nfi_synth.h).
//
// Data layout.  Activations are channel-last ([B,H,W,C]) and exist as a PAIR of bf16 tensors,
// hi = bf16(value) and lo = bf16(value - hi) (16 significant bits between them, 4 bytes per element
// like the fp32 they stand for), already multiplied by the style of the layer that will consume
// them (conv_modulated2d scales the activations, not the weights: stylegan.py:131).  Weights are
// re-laid-out per call to [tap][Cout][Cin] (K-major rows for the B operand), also as hi / lo.  One
// 3x3 tap of one 64-channel block is then ONE TMA box per operand: a [1 x 8 x 16 x 64] box of the
// activation tensor at the tile origin shifted by the tap (out-of-range rows / columns / channels
// arrive as zeros = the conv padding) is a 256-row x 128-byte SWIZZLE_128B tile = the K-major A
// operand of four 64 x BN x 64 wgmma row blocks; no im2col buffer, no register staging.  D
// accumulates over taps x channel blocks in registers as A_lo W_hi + A_hi W_lo + A_hi W_hi (bf16
// operands, fp32 accumulate): the dropped lo x lo term is 2^-18 of a product.  (3xTF32 on fp32
// pairs would double the tensor time for operands exact to 2^-22 without a more accurate result:
// the tensor core adds the products of one output into its fp32 accumulator with truncation, and
// that bias, which grows with K, dominates either way.)
//
// conv_tc_kernel (persistent, 384 threads):
//   warpgroup 0    TMA producer : 4 boxes per k-iteration (A_hi, A_lo 32 KB each, W_hi, W_lo) into a
//                                 2-stage ring (one elected thread)
//   warpgroups 1-2 consumers    : rows 128c .. 128c + 127 of the position tile as two 64-row wgmma
//                                 blocks, 24 wgmma (bf16, M64 N<=128 K16) per stage, the stage released
//                                 once the next one's are in flight; then the fused epilogue straight
//                                 from the accumulator registers -> global
// Epilogues: ACT  x*dcoef + noise + bias, *sqrt(2), leaky-relu 0.2, then for up to two consumers
//                 (next conv, ToRGB) * their style -> hi / lo           (stylegan.py:137-142,349-356)
//            RAW  plain store at (2a+py, 2b+px) of the (2H+1)x(2W+1) transposed-conv result; the
//                 stride-2 transposed convolution (stylegan.py:98-100) is four such phase GEMMs over
//                 the INPUT grid (4 + 2 + 2 + 1 taps), then fir_act_kernel applies the 4x4 FIR
//                 (gain 4, pad 1, stylegan.py:101) and the ACT epilogue
//            RGB  ToRGB: + bias + FIR-upsampled running image (stylegan.py:71-75,430-433); the
//                 last block writes the tri-planes channel-last [B,3,R,R,32]
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "nfi_synth.h"
#include "nfi_synth_launch.h"
#include "nfi_tc.cuh"

namespace nfi {
namespace synth {

constexpr int kTileH = 16, kTileW = 16;  // 256 output positions = four wgmma M = 64 blocks
constexpr int kKBlock = 64;             // bf16 channels per k-iteration: 128-byte rows
constexpr int kStages = 2;
constexpr int kATile = 256 * 128;       // bytes of one A box: 256 rows of 128 bytes
constexpr int kConvThreads = 384;      // TMA warpgroup, two consumer warpgroups
constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // 384 x 168 = 128 x (40 + 2 x 232) + 512
constexpr int kMaxPhases = 4, kMaxTaps = 9;

enum { kModeRaw = 0, kModeAct = 1, kModeRgb = 2 };
// ToRGB: the running image's footprint of one 16x16 output tile is 10x10 low-resolution positions
// x 96 channels; staged once per tile in shared memory (rows padded to 25 float4: consecutive
// positions fall into different bank groups)
constexpr int kSkipDim = 10, kSkipRow4 = 25;
constexpr int kSkipBytes = kSkipDim * kSkipDim * kSkipRow4 * 16;

struct ActEpilogue {   // shared by conv_tc_kernel (stride-1 layers) and fir_act_kernel (up layers)
  const float* dcoef;  // [B,N]
  const float* noise;  // [B,H,W] or nullptr
  const float* bias;   // [N]
  float gain;          // sqrt(2)
  const float* style_a;  // [B,N] style of consumer a (or nullptr: plain value)
  __nv_bfloat16* a_hi;   // [B,H,W,N]
  __nv_bfloat16* a_lo;
  const float* style_b;  // second consumer or nullptr
  __nv_bfloat16* b_hi;
  __nv_bfloat16* b_lo;
  float* u_out;          // [B,H,W,N] pre-activation u for the backward, or nullptr (plain forward)
};

struct ConvArgs {
  int B, C, N, BN, n_tiles_n;
  int H, W;  // extent of the input tensor (= extent of the output for stride-1 layers)
  int n_phases;
  int ph_taps[kMaxPhases];      // taps of the phase
  int ph_tap0[kMaxPhases];      // first entry in tap_* of the phase
  int ph_DH[kMaxPhases], ph_DW[kMaxPhases];        // domain of the phase (rows, cols)
  int ph_ty[kMaxPhases], ph_tx[kMaxPhases];        // tiles
  int ph_tile0[kMaxPhases + 1];                    // first m-tile of the phase (per image count)
  int ph_oy[kMaxPhases], ph_ox[kMaxPhases];        // RAW: output offset of the phase
  int tap_dy[kMaxTaps], tap_dx[kMaxTaps], tap_w[kMaxTaps];
  int tap_img[kMaxTaps];        // image offset of the tap's A box (backward phase maps; else 0)
  int mode;
  // RAW
  float* out_raw;
  int out_H, out_W, out_stride;  // output extent, position stride (2 for the transposed conv)
  // ACT
  ActEpilogue act;
  // RGB
  const float* skip;  // [B,H/2,W/2,N] running image of the previous block or nullptr
  float* img;         // [B,H,W,N] or nullptr
  float* planes;      // [B,3,H,W,32] or nullptr (last block)
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2,
                                            int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(tc::smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(tc::smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3, %4}], [%5];" ::"r"(tc::smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(tc::smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc::smem_u32(bar)) : "memory");
}

struct TileCoord {
  int phase, img, ty, tx, nt;
};
__device__ __forceinline__ TileCoord decode_tile(const ConvArgs& a, int tile) {
  TileCoord t;
  t.nt = tile % a.n_tiles_n;  // the n-tiles of one position tile run back to back: A stays in L2
  int m = tile / a.n_tiles_n;
  const int per_img = a.ph_tile0[a.n_phases];
  t.img = m / per_img;
  m -= t.img * per_img;
  t.phase = 0;
#pragma unroll
  for (int p = 1; p < kMaxPhases; ++p)
    if (p < a.n_phases && m >= a.ph_tile0[p]) t.phase = p;
  m -= a.ph_tile0[t.phase];
  t.ty = m / a.ph_tx[t.phase];
  t.tx = m - t.ty * a.ph_tx[t.phase];
  return t;
}

// t = hi + lo with hi = bf16(t), lo = bf16(t - hi)
__device__ __forceinline__ void split_bf16(float t, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(t);
  lo = __float2bfloat16_rn(t - __bfloat162float(hi));
}
// value -> (value * style) as a bf16 hi / lo pair, 4 channels (8 bytes per tensor) at a time
__device__ __forceinline__ void store_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t idx,
                                             float4 v, float4 s) {
  __align__(8) __nv_bfloat16 h[4], l[4];
  split_bf16(v.x * s.x, h[0], l[0]);
  split_bf16(v.y * s.y, h[1], l[1]);
  split_bf16(v.z * s.z, h[2], l[2]);
  split_bf16(v.w * s.w, h[3], l[3]);
  *reinterpret_cast<uint2*>(hi + idx) = *reinterpret_cast<const uint2*>(h);
  *reinterpret_cast<uint2*>(lo + idx) = *reinterpret_cast<const uint2*>(l);
}
__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : 0.2f * x; }

// value -> (value * style) as a bf16 hi / lo pair, 2 channels (4 bytes per tensor) at a time
__device__ __forceinline__ void store_split2(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t idx,
                                             float2 v, float2 s) {
  __align__(4) __nv_bfloat16 h[2], l[2];
  split_bf16(v.x * s.x, h[0], l[0]);
  split_bf16(v.y * s.y, h[1], l[1]);
  *reinterpret_cast<uint32_t*>(hi + idx) = *reinterpret_cast<const uint32_t*>(h);
  *reinterpret_cast<uint32_t*>(lo + idx) = *reinterpret_cast<const uint32_t*>(l);
}
// The ACT epilogue on 2 consecutive channels n, n+1 of position `pos` (the conv kernel's register
// fragments hold channel pairs).
__device__ __forceinline__ void act_store2(const ActEpilogue& e, int img, size_t pos, int N, int n,
                                           float2 acc, float noise) {
  const float2 d = __ldg(reinterpret_cast<const float2*>(e.dcoef + (size_t)img * N + n));
  const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + n));
  float2 u, v;
  u.x = ((acc.x * d.x + noise) + b.x) * e.gain;
  u.y = ((acc.y * d.y + noise) + b.y) * e.gain;
  if (e.u_out != nullptr) *reinterpret_cast<float2*>(e.u_out + pos * N + n) = u;
  v.x = lrelu(u.x);
  v.y = lrelu(u.y);
  const float2 one = make_float2(1.f, 1.f);
  if (e.a_hi != nullptr) {
    const float2 s = e.style_a ? __ldg(reinterpret_cast<const float2*>(e.style_a + (size_t)img * N + n)) : one;
    store_split2(e.a_hi, e.a_lo, pos * N + n, v, s);
  }
  if (e.b_hi != nullptr) {
    const float2 s = e.style_b ? __ldg(reinterpret_cast<const float2*>(e.style_b + (size_t)img * N + n)) : one;
    store_split2(e.b_hi, e.b_lo, pos * N + n, v, s);
  }
}
// The ACT epilogue on 4 consecutive channels n..n+3 of position `pos` (= (img*H + y)*W + x).
__device__ __forceinline__ void act_store4(const ActEpilogue& e, int img, size_t pos, int N, int n,
                                           float4 acc, float noise) {
  const float4 d = __ldg(reinterpret_cast<const float4*>(e.dcoef + (size_t)img * N + n));
  const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + n));
  float4 u, v;
  u.x = ((acc.x * d.x + noise) + b.x) * e.gain;
  u.y = ((acc.y * d.y + noise) + b.y) * e.gain;
  u.z = ((acc.z * d.z + noise) + b.z) * e.gain;
  u.w = ((acc.w * d.w + noise) + b.w) * e.gain;
  if (e.u_out != nullptr) *reinterpret_cast<float4*>(e.u_out + pos * N + n) = u;
  v.x = lrelu(u.x);
  v.y = lrelu(u.y);
  v.z = lrelu(u.z);
  v.w = lrelu(u.w);
  const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
  if (e.a_hi != nullptr) {
    const float4 s = e.style_a ? __ldg(reinterpret_cast<const float4*>(e.style_a + (size_t)img * N + n)) : one;
    store_split4(e.a_hi, e.a_lo, pos * N + n, v, s);
  }
  if (e.b_hi != nullptr) {
    const float4 s = e.style_b ? __ldg(reinterpret_cast<const float4*>(e.style_b + (size_t)img * N + n)) : one;
    store_split4(e.b_hi, e.b_lo, pos * N + n, v, s);
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t a, uint64_t b) {
  if constexpr (BN == 32) tc::wgmma_bf16_ss_n32<0, 0>(d, a, b, 1);
  else if constexpr (BN == 64) tc::wgmma_bf16_ss_n64<0, 0>(d, a, b, 1);
  else if constexpr (BN == 96) tc::wgmma_bf16_ss_n96<0, 0>(d, a, b, 1);
  else tc::wgmma_bf16_ss_n128<0, 0>(d, a, b, 1);
}

// Consumer warpgroup c (0, 1): rows 128c .. 128c + 127 of each position tile, BN columns.
template <int BN>
__device__ __forceinline__ void conv_consume(const ConvArgs& a, int n_tiles, unsigned char* smem,
                                             uint64_t* full, uint64_t* empty, float4* skip_sm,
                                             int c, int ctid) {
  const int lane = ctid & 31, warp = ctid >> 5 & 3;
  const int g4 = lane >> 2, t = lane & 3;
  const int w_tile = BN * 128;
  const int stage_bytes = 2 * kATile + 2 * w_tile;
  const int kblocks = (a.C + kKBlock - 1) / kKBlock;  // a partial last block is zero-filled by TMA
  const uint32_t smem_s = tc::smem_u32(smem);
  uint32_t st = 0, ph = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const TileCoord tl = decode_tile(a, tile);
    const int n0 = tl.nt * BN;
    const bool staged = (a.mode == kModeRgb) && (a.skip != nullptr);
    if (staged) {
      // before the MMAs of this tile: the 10x10 low-resolution footprint of the tile, zeros
      // outside the image (a missing neighbour contributes nothing, stylegan.py:71-75)
      const int hh = a.H >> 1, hw = a.W >> 1;
      const int gy0 = tl.ty * (kTileH / 2) - 1, gx0 = tl.tx * (kTileW / 2) - 1;
      const int c4n = a.N >> 2;   // float4 per position (24)
      tc::bar_sync(1, 256);       // the previous tile's readers are done
      for (int i = ctid; i < kSkipDim * kSkipDim * c4n; i += 256) {
        const int pxl = i / c4n, c4 = i - pxl * c4n;
        const int gy = gy0 + pxl / kSkipDim, gx = gx0 + pxl % kSkipDim;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gy >= 0 && gy < hh && gx >= 0 && gx < hw)
          v = __ldg(reinterpret_cast<const float4*>(a.skip + (((size_t)tl.img * hh + gy) * hw + gx) * a.N) + c4);
        skip_sm[pxl * kSkipRow4 + c4] = v;
      }
      tc::bar_sync(1, 256);
    }
    float acc[2][BN / 2];
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[mb][i] = 0.f;
    tc::wgmma_fence();
    const int iters = a.ph_taps[tl.phase] * kblocks;
    uint32_t prev_st = 0;
    for (int k = 0; k < iters; ++k) {
      tc::mbar_wait(&full[st], ph);
      const uint32_t sb = smem_s + st * stage_bytes;
      const uint64_t w_hi = tc::gmma_desc_sw128(sb + 2 * kATile);
      const uint64_t w_lo = tc::gmma_desc_sw128(sb + 2 * kATile + w_tile);
      // the W boxes of the stage serve both row blocks of this warpgroup
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        const uint32_t rows = (uint32_t)(128 * c + 64 * mb) * 128;
        const uint64_t a_hi = tc::gmma_desc_sw128(sb + rows);
        const uint64_t a_lo = tc::gmma_desc_sw128(sb + kATile + rows);
        // small terms first; a K step of 16 bf16 = 32 bytes = +2 in the descriptor's address field
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_bn<BN>(acc[mb], a_lo + 2 * ks, w_hi + 2 * ks);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_bn<BN>(acc[mb], a_hi + 2 * ks, w_lo + 2 * ks);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_bn<BN>(acc[mb], a_hi + 2 * ks, w_hi + 2 * ks);
      }
      tc::wgmma_commit();
      // the previous stage's products are complete once at most this one's are in flight
      tc::wgmma_wait<1>();
      if (k > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev_st]);
      }
      prev_st = st;
      if (++st == kStages) { st = 0; ph ^= 1; }
    }
    tc::wgmma_wait<0>();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) tc::reg_fence(acc[mb]);
    __syncwarp();
    if (iters > 0 && lane == 0) mbar_arrive(&empty[prev_st]);

    // ================================ EPILOGUE ================================
    const float* skipf = reinterpret_cast<const float*>(skip_sm);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = 128 * c + 64 * mb + 16 * warp + g4 + 8 * half;  // position (row / 16, row % 16)
        const int y = tl.ty * kTileH + row / kTileW, x = tl.tx * kTileW + row % kTileW;
        const bool valid = (y < a.ph_DH[tl.phase]) && (x < a.ph_DW[tl.phase]);
        if (!valid) continue;
        float noise = 0.f;
        size_t pos = 0;
        float wsk[4] = {0.f, 0.f, 0.f, 0.f};
        int psk[4] = {0, 0, 0, 0};
        if (a.mode == kModeRaw) {
          const int oy = a.out_stride * y + a.ph_oy[tl.phase], ox = a.out_stride * x + a.ph_ox[tl.phase];
          pos = ((size_t)tl.img * a.out_H + oy) * a.out_W + ox;
        } else {
          pos = ((size_t)tl.img * a.H + y) * a.W + x;
          if (a.mode == kModeAct && a.act.noise != nullptr) noise = __ldg(a.act.noise + pos);
          if (staged) {
            // upsample2d (stylegan.py:71-75): out[2i] = 3/4 in[i] + 1/4 in[i-1], out[2i+1] = 3/4 in[i]
            // + 1/4 in[i+1] per axis; positions inside the staged footprint (its origin is one
            // low-res position up / left of the tile); out-of-image neighbours are staged as zeros,
            // so the weights need no masking
            const int iy = y >> 1, ix = x >> 1;
            const int jy = (y & 1) ? iy + 1 : iy - 1, jx = (x & 1) ? ix + 1 : ix - 1;
            const int ly = iy - (tl.ty * (kTileH / 2) - 1), lx = ix - (tl.tx * (kTileW / 2) - 1);
            const int my = jy - (tl.ty * (kTileH / 2) - 1), mx = jx - (tl.tx * (kTileW / 2) - 1);
            wsk[0] = 0.75f * 0.75f; psk[0] = ly * kSkipDim + lx;
            wsk[1] = 0.75f * 0.25f; psk[1] = ly * kSkipDim + mx;
            wsk[2] = 0.25f * 0.75f; psk[2] = my * kSkipDim + lx;
            wsk[3] = 0.25f * 0.25f; psk[3] = my * kSkipDim + mx;
          }
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          float2 v = make_float2(acc[mb][4 * j + 2 * half], acc[mb][4 * j + 2 * half + 1]);
          const int nn = n0 + 8 * j + 2 * t;
          if (a.mode == kModeRaw) {
            *reinterpret_cast<float2*>(a.out_raw + pos * a.N + nn) = v;
          } else if (a.mode == kModeAct) {
            act_store2(a.act, tl.img, pos, a.N, nn, v, noise);
          } else {
            const float2 b = __ldg(reinterpret_cast<const float2*>(a.act.bias + nn));
            v.x += b.x;
            v.y += b.y;
            if (staged) {
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float2 k2 = *reinterpret_cast<const float2*>(skipf + (psk[q] * kSkipRow4) * 4 + nn);
                v.x = fmaf(wsk[q], k2.x, v.x);
                v.y = fmaf(wsk[q], k2.y, v.y);
              }
            }
            if (a.img != nullptr) *reinterpret_cast<float2*>(a.img + pos * a.N + nn) = v;
            if (a.planes != nullptr) {
              const int pl = nn >> 5, ch = nn & 31;
              const size_t o = ((((size_t)tl.img * 3 + pl) * a.H + y) * a.W + x) * 32 + ch;
              *reinterpret_cast<float2*>(a.planes + o) = v;
            }
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kConvThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
               const __grid_constant__ ConvArgs a, int n_tiles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const int w_tile = a.BN * 128;                 // bytes of one W box
  const int stage_bytes = 2 * kATile + 2 * w_tile;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * stage_bytes);
  uint64_t* full = bars;                // [kStages] TMA landed
  uint64_t* empty = full + kStages;     // [kStages] wgmma of the stage complete (8 consumer warps)
  float4* skip_sm = reinterpret_cast<float4*>(smem + kStages * stage_bytes + 128);  // RGB + skip only

  if (tid == 0) {
    if (tc::smem_u32(smem) & 1023u) __trap();
    for (int i = 0; i < kStages; ++i) {
      tc::mbar_init(&full[i], 1);
      tc::mbar_init(&empty[i], 8);
    }
    tc::fence_mbar_init();
    prefetch_tmap(&tmAh);
    prefetch_tmap(&tmAl);
    prefetch_tmap(&tmWh);
    prefetch_tmap(&tmWl);
  }
  __syncthreads();
  const int kblocks = (a.C + kKBlock - 1) / kKBlock;  // a partial last block is zero-filled by TMA

  if (wg == 0) {
    // ================================ TMA PRODUCER ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (tid < 32 && elect_one()) {
      uint32_t st = 0, ph = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const TileCoord t = decode_tile(a, tile);
        const int y0 = t.ty * kTileH, x0 = t.tx * kTileW, n0 = t.nt * a.BN;
        const int tap0 = a.ph_tap0[t.phase];
        for (int tp = 0; tp < a.ph_taps[t.phase]; ++tp) {
          const int dy = a.tap_dy[tap0 + tp], dx = a.tap_dx[tap0 + tp], tw = a.tap_w[tap0 + tp];
          const int im = t.img + a.tap_img[tap0 + tp];
          for (int kb = 0; kb < kblocks; ++kb) {
            tc::mbar_wait(&empty[st], ph ^ 1);
            unsigned char* s = smem + st * stage_bytes;
            tc::mbar_expect_tx(&full[st], (uint32_t)stage_bytes);
            tma_load_4d(s, &tmAh, kb * kKBlock, x0 + dx, y0 + dy, im, &full[st]);
            tma_load_4d(s + kATile, &tmAl, kb * kKBlock, x0 + dx, y0 + dy, im, &full[st]);
            tma_load_3d(s + 2 * kATile, &tmWh, kb * kKBlock, n0, tw, &full[st]);
            tma_load_3d(s + 2 * kATile + w_tile, &tmWl, kb * kKBlock, n0, tw, &full[st]);
            if (++st == kStages) { st = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    // ================================ CONSUMERS ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int c = wg - 1, ctid = tid - 128;
    switch (a.BN) {
      case 32: conv_consume<32>(a, n_tiles, smem, full, empty, skip_sm, c, ctid); break;
      case 64: conv_consume<64>(a, n_tiles, smem, full, empty, skip_sm, c, ctid); break;
      case 96: conv_consume<96>(a, n_tiles, smem, full, empty, skip_sm, c, ctid); break;
      default: conv_consume<128>(a, n_tiles, smem, full, empty, skip_sm, c, ctid); break;
    }
  }
}

// 4x4 FIR (outer([1,3,3,1]) / 16 = the reference's filter * gain 4, pad 1) over the (2H+1)x(2W+1)
// transposed-conv result, then the ACT epilogue.  One thread per (2x2 output block, 4 channels):
// the block needs a 5x5 window of the raw tensor (25 loads for 4 outputs instead of 16 each), rows
// filtered first (separable), then columns.
__global__ void __launch_bounds__(256)
fir_act_kernel(const float* __restrict__ raw, int B, int OH, int OW, int N, ActEpilogue e) {
  const int RH = OH + 1, RW = OW + 1;
  const int groups = N >> 2, bh = OH >> 1, bw = OW >> 1;
  const size_t total = (size_t)B * bh * bw * groups;
  const float kf[4] = {0.25f, 0.75f, 0.75f, 0.25f};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const size_t blk = i / groups;
    const int v0 = 2 * (int)(blk % bw);
    const int u0 = 2 * (int)((blk / bw) % bh);
    const int img = (int)(blk / ((size_t)bw * bh));
    // horizontally filtered rows u0-1 .. u0+3 for the two output columns v0, v0+1
    float4 h0[5], h1[5];
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const int ry = u0 + r - 1;
      float4 t[5];
#pragma unroll
      for (int c = 0; c < 5; ++c) {
        const int rx = v0 + c - 1;
        t[c] = (ry >= 0 && ry < RH && rx >= 0 && rx < RW)
                   ? __ldg(reinterpret_cast<const float4*>(raw + (((size_t)img * RH + ry) * RW + rx) * N + 4 * g))
                   : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#define NFI_H(cmp)                                                                              \
  h0[r].cmp = fmaf(kf[3], t[3].cmp, fmaf(kf[2], t[2].cmp, fmaf(kf[1], t[1].cmp, kf[0] * t[0].cmp))); \
  h1[r].cmp = fmaf(kf[3], t[4].cmp, fmaf(kf[2], t[3].cmp, fmaf(kf[1], t[2].cmp, kf[0] * t[1].cmp)));
      NFI_H(x) NFI_H(y) NFI_H(z) NFI_H(w)
#undef NFI_H
    }
#pragma unroll
    for (int du = 0; du < 2; ++du) {
#pragma unroll
      for (int dv = 0; dv < 2; ++dv) {
        const float4* hh = dv ? h1 : h0;
        float4 acc;
#define NFI_V(cmp)                                                                  \
  acc.cmp = fmaf(kf[3], hh[du + 3].cmp,                                             \
                 fmaf(kf[2], hh[du + 2].cmp, fmaf(kf[1], hh[du + 1].cmp, kf[0] * hh[du].cmp)));
        NFI_V(x) NFI_V(y) NFI_V(z) NFI_V(w)
#undef NFI_V
        const size_t pos = ((size_t)img * OH + (u0 + du)) * OW + (v0 + dv);
        const float noise = e.noise ? __ldg(e.noise + pos) : 0.f;
        act_store4(e, img, pos, N, 4 * g, acc, noise);
      }
    }
  }
}

// weight [Cout,Cin,K,K] -> [K*K][Cout][Cin] hi / lo (K-major rows of the B operand) and
// wsq[Cout][Cin] = sum over taps of W^2 (for the demodulation coefficients)
__global__ void prep_weights_kernel(const float* __restrict__ w, int cout, int cin, int taps,
                                    __nv_bfloat16* __restrict__ w_hi,
                                    __nv_bfloat16* __restrict__ w_lo, float* __restrict__ wsq) {
  const size_t total = (size_t)cout * cin;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    float sq = 0.f;
    for (int t = 0; t < taps; ++t) {
      const float v = w[i * taps + t];
      split_bf16(v, w_hi[(size_t)t * total + i], w_lo[(size_t)t * total + i]);
      sq = fmaf(v, v, sq);
    }
    if (wsq != nullptr) wsq[i] = sq;
  }
}

// styles[b,c] = (affine_w[c,:] . w[b,:] / sqrt(w_dim) + affine_b[c]) * gain   (stylegan.py:148-180,
// 329,372); one warp per (b, c)
__global__ void styles_kernel(const float* __restrict__ ws, int ws_stride, int w_dim,
                              const float* __restrict__ aw, const float* __restrict__ ab, int cin,
                              int B, float gain, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * cin) return;
  const int b = warp / cin, c = warp % cin;
  const float* wv = ws + (size_t)b * ws_stride;
  const float* row = aw + (size_t)c * w_dim;
  float s = 0.f;
  for (int k = lane; k < w_dim; k += 32) s = fmaf(row[k], wv[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[warp] = (s * rsqrtf((float)w_dim) + ab[c]) * gain;
}

// dcoef[b,o] = rsqrt(sum_c wsq[o,c] s[b,c]^2 + 1e-8)  (stylegan.py:128); one warp per (b, o)
__global__ void dcoef_kernel(const float* __restrict__ wsq, const float* __restrict__ s, int cout,
                             int cin, int B, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * cout) return;
  const int b = warp / cout, o = warp % cout;
  float acc = 0.f;
  for (int c = lane; c < cin; c += 32) {
    const float sv = s[(size_t)b * cin + c];
    acc = fmaf(wsq[(size_t)o * cin + c], sv * sv, acc);
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, k);
  if (lane == 0) out[warp] = rsqrtf(acc + 1e-8f);
}

// b4.const [C,4,4] repeated over the batch (stylegan.py:422), scaled by conv1's style -> hi / lo
__global__ void const_input_kernel(const float* __restrict__ cst, const float* __restrict__ style,
                                   int B, int C, __nv_bfloat16* __restrict__ hi,
                                   __nv_bfloat16* __restrict__ lo) {
  const int total = B * 16 * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % C, p = (i / C) % 16, b = i / (16 * C);
    split_bf16(cst[c * 16 + p] * style[b * C + c], hi[i], lo[i]);
  }
}

// ------------------------------------------------------------------ backward to the latents
// The data gradients dx~ = conv^T(dacc, W) run on conv_tc_kernel (RAW mode) with the weights
// re-laid-out below; everything between two GEMMs of a layer is ONE full-resolution pass
// (act_backward_kernel), plus the FIR adjoint for the up layers.

// weight [Cout,Cin,K,K] -> [K*K][Cin][Cout] hi / lo: the B operand of the data-gradient GEMM
// (reduction over Cout).  The stride-1 layer's tap flip lives in the tap table, not here.
__global__ void prep_weights_t_kernel(const float* __restrict__ w, int cout, int cin, int taps,
                                      __nv_bfloat16* __restrict__ w_hi,
                                      __nv_bfloat16* __restrict__ w_lo) {
  const size_t total = (size_t)cout * cin;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t ci = i / cout, o = i - ci * cout;   // output index (ci, o): o fastest
    for (int t = 0; t < taps; ++t)
      split_bf16(w[(o * cin + ci) * taps + t], w_hi[(size_t)t * total + i], w_lo[(size_t)t * total + i]);
  }
}

struct ActBackward {
  const float* u;       // [B,HW,C] saved pre-activation of the layer
  const float* noise;   // [B,HW] or nullptr
  const float* bias;    // [C]
  const float* dcoef;   // [B,C]
  float gain;           // sqrt(2)
  // up to two consumers of v = lrelu(u): the gradient of their STYLED input (dx~), their style s,
  // and ds[b,c] += sum_pos dx~ v (the data half of their style gradient)
  const float* dx_a; const float* s_a; float* ds_a;
  const float* dx_b; const float* s_b; float* ds_b;
  float* dd;            // [B,C] += sum_pos g (acc d),  g = dv lrelu'(u) gain
  __nv_bfloat16* dacc_hi;  // dacc = g d as a pair (input of the next data-gradient GEMM) ...
  __nv_bfloat16* dacc_lo;
  float* dacc;             // ... or fp32 (input of the FIR adjoint)
};

__device__ __forceinline__ float lrelu_grad(float u) { return u > 0.f ? 1.f : 0.2f; }

// One pass over a layer's output: dv = dx~_a s_a + dx~_b s_b, then dacc = dv lrelu'(u) gain d, and
// the per-(b, channel) sums ds_a, ds_b, dd.  Block (chunk, b): 4 channels per thread, 256 / (C/4)
// positions in parallel; the sums are reduced in shared memory, then one atomic per block.
__global__ void __launch_bounds__(256)
act_backward_kernel(ActBackward e, int HW, int C, int chunk) {
  __shared__ float4 red[3][256];
  const int cg = C >> 2, ppar = 256 / cg, tid = threadIdx.x;
  const int p = tid / cg, c4 = tid - p * cg;
  const int b = blockIdx.y;
  const bool active = p < ppar;
  const float inv_gain = 1.f / e.gain;
  float4 sa = make_float4(0.f, 0.f, 0.f, 0.f), sb = sa, sd = sa;
  if (active) {
    const float4 d = *reinterpret_cast<const float4*>(e.dcoef + (size_t)b * C + 4 * c4);
    const float4 bi = *reinterpret_cast<const float4*>(e.bias + 4 * c4);
    const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 s_a = e.s_a ? *reinterpret_cast<const float4*>(e.s_a + (size_t)b * C + 4 * c4) : one;
    const float4 s_b = e.s_b ? *reinterpret_cast<const float4*>(e.s_b + (size_t)b * C + 4 * c4) : one;
    const int end = min(HW, (blockIdx.x + 1) * chunk);
    for (int pos = blockIdx.x * chunk + p; pos < end; pos += ppar) {
      const size_t row = (size_t)b * HW + pos, idx = row * C + 4 * c4;
      const float4 u = __ldg(reinterpret_cast<const float4*>(e.u + idx));
      const float nz = e.noise ? __ldg(e.noise + row) : 0.f;
      float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
#define NFI_CONSUMER(dx, s, acc)                                                    \
  if (dx != nullptr) {                                                              \
    const float4 x = __ldg(reinterpret_cast<const float4*>(dx + idx));              \
    acc.x = fmaf(x.x, lrelu(u.x), acc.x); acc.y = fmaf(x.y, lrelu(u.y), acc.y);     \
    acc.z = fmaf(x.z, lrelu(u.z), acc.z); acc.w = fmaf(x.w, lrelu(u.w), acc.w);     \
    dv.x = fmaf(x.x, s.x, dv.x); dv.y = fmaf(x.y, s.y, dv.y);                       \
    dv.z = fmaf(x.z, s.z, dv.z); dv.w = fmaf(x.w, s.w, dv.w);                       \
  }
      NFI_CONSUMER(e.dx_a, s_a, sa)
      NFI_CONSUMER(e.dx_b, s_b, sb)
#undef NFI_CONSUMER
      float4 g, out;
#define NFI_G(cmp)                                                                   \
  g.cmp = dv.cmp * lrelu_grad(u.cmp) * e.gain;                                       \
  sd.cmp = fmaf(g.cmp, u.cmp * inv_gain - nz - bi.cmp, sd.cmp);  /* acc d = u/gain - noise - bias */ \
  out.cmp = g.cmp * d.cmp;
      NFI_G(x) NFI_G(y) NFI_G(z) NFI_G(w)
#undef NFI_G
      if (e.dacc_hi != nullptr) store_split4(e.dacc_hi, e.dacc_lo, idx, out, one);
      if (e.dacc != nullptr) *reinterpret_cast<float4*>(e.dacc + idx) = out;
    }
  }
  red[0][tid] = sa;
  red[1][tid] = sb;
  red[2][tid] = sd;
  __syncthreads();
  if (tid < cg) {
    float* dst[3] = {e.ds_a, e.ds_b, e.dd};
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      if (dst[q] == nullptr) continue;
      float4 s = red[q][tid];
      for (int k = 1; k < ppar; ++k) {
        const float4 t = red[q][k * cg + tid];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      float* o = dst[q] + (size_t)b * C + 4 * tid;
      atomicAdd(o + 0, s.x);
      atomicAdd(o + 1, s.y);
      atomicAdd(o + 2, s.z);
      atomicAdd(o + 3, s.w);
    }
  }
}

// Adjoint of the up layer's 4x4 FIR (symmetric, so a correlation with the same taps), written as
// the four parity phases of the (2H+1)^2 raw gradient: phase (py,px) at image offset (2py+px)*B of
// a [4B, H+1, W+1, C] pair, position (a,b) = raw (2a+py, 2b+px); entries past the raw extent are 0.
__global__ void fir_adjoint_kernel(const float* __restrict__ dacc, int B, int OH, int OW, int C,
                                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int PH = OH / 2 + 1, PW = OW / 2 + 1, groups = C >> 2;
  const size_t total = (size_t)4 * B * PH * PW * groups;
  const float kf[4] = {0.25f, 0.75f, 0.75f, 0.25f};
  const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    size_t r = i / groups;
    const int bx = (int)(r % PW); r /= PW;
    const int ay = (int)(r % PH); r /= PH;
    const int img = (int)(r % B);
    const int phase = (int)(r / B);
    const int ry = 2 * ay + (phase >> 1), rx = 2 * bx + (phase & 1);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ry <= OH && rx <= OW) {
#pragma unroll
      for (int ka = 0; ka < 4; ++ka) {
        const int y = ry - ka + 1;
        if (y < 0 || y >= OH) continue;
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
          const int x = rx - kb + 1;
          if (x < 0 || x >= OW) continue;
          const float w = kf[ka] * kf[kb];
          const float4 t = __ldg(reinterpret_cast<const float4*>(dacc + (((size_t)img * OH + y) * OW + x) * C) + g);
          acc.x = fmaf(w, t.x, acc.x); acc.y = fmaf(w, t.y, acc.y);
          acc.z = fmaf(w, t.z, acc.z); acc.w = fmaf(w, t.w, acc.w);
        }
      }
    }
    store_split4(hi, lo, i * 4, acc, one);
  }
}

// d(planes) [B,3,R,R,32] -> d(image) [B,R,R,96] (channel nn = plane * 32 + c), fp32 and as a pair
__global__ void planes_grad_kernel(const float* __restrict__ gp, int B, int R, float* __restrict__ out,
                                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const size_t total = (size_t)B * R * R * 96;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i % 96);
    const size_t pix = i / 96, img = pix / ((size_t)R * R), yx = pix - img * R * R;
    const float v = gp[((img * 3 + nn / 32) * R * R + yx) * 32 + (nn & 31)];
    out[i] = v;
    split_bf16(v, hi[i], lo[i]);
  }
}

// Adjoint of upsample_img (stylegan.py:71-75) per axis: din[i] = 3/4 (dout[2i] + dout[2i+1]) +
// 1/4 (dout[2i-1] + dout[2i+2]); [B,2h,2w,C] -> [B,h,w,C], fp32 and as a pair
__global__ void upsample_adjoint_kernel(const float* __restrict__ dout, int B, int h, int w, int C,
                                        float* __restrict__ out, __nv_bfloat16* __restrict__ hi,
                                        __nv_bfloat16* __restrict__ lo) {
  const size_t total = (size_t)B * h * w * C;
  const float kf[4] = {0.25f, 0.75f, 0.75f, 0.25f};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int x = (int)(r % w); r /= w;
    const int y = (int)(r % h);
    const int img = (int)(r / h);
    float acc = 0.f;
    for (int a = 0; a < 4; ++a) {
      const int Y = 2 * y - 1 + a;
      if (Y < 0 || Y >= 2 * h) continue;
      for (int bb = 0; bb < 4; ++bb) {
        const int X = 2 * x - 1 + bb;
        if (X < 0 || X >= 2 * w) continue;
        acc = fmaf(kf[a] * kf[bb], dout[(((size_t)img * 2 * h + Y) * 2 * w + X) * C + c], acc);
      }
    }
    out[i] = acc;
    split_bf16(acc, hi[i], lo[i]);
  }
}

// The demodulation chain: d = rsqrt(sum_o' wsq s^2 + 1e-8) gives dd/ds_i = -d^3 wsq[o,i] s_i, and
// dd_true = dd_part / d (act_backward_kernel sums g (acc d)), so
// ds[b,i] -= s_i sum_o dd_part[b,o] d[b,o]^2 wsq[o,i]; one warp per (b, i)
__global__ void dcoef_backward_kernel(const float* __restrict__ wsq, const float* __restrict__ s,
                                      const float* __restrict__ dd, const float* __restrict__ d,
                                      int cout, int cin, int B, float* __restrict__ ds) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * cin) return;
  const int b = warp / cin, i = warp % cin;
  float acc = 0.f;
  for (int o = lane; o < cout; o += 32) {
    const float dv = d[(size_t)b * cout + o];
    acc = fmaf(dd[(size_t)b * cout + o] * dv * dv, wsq[(size_t)o * cin + i], acc);
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, k);
  if (lane == 0) ds[warp] -= s[warp] * acc;
}

// block 0's conv1 reads b4.const * style: ds[b,c] += sum_p dx~[b,p,c] const[c,p]
__global__ void const_ds_kernel(const float* __restrict__ dx, const float* __restrict__ cst, int B,
                                int C, float* __restrict__ ds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i % C;
  float acc = 0.f;
  for (int p = 0; p < 16; ++p) acc = fmaf(dx[((size_t)b * 16 + p) * C + c], cst[c * 16 + p], acc);
  ds[i] += acc;
}

// The transpose of styles_kernel: g_ws[b,row,k] += gain / sqrt(w_dim) sum_c ds[b,c] A[c,k]
__global__ void styles_backward_kernel(const float* __restrict__ ds, const float* __restrict__ aw,
                                       int cin, int w_dim, int B, float scale, float* __restrict__ g_ws,
                                       int ws_stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * w_dim) return;
  const int b = i / w_dim, k = i % w_dim;
  float acc = 0.f;
  for (int c = 0; c < cin; ++c) acc = fmaf(ds[(size_t)b * cin + c], aw[(size_t)c * w_dim + k], acc);
  g_ws[(size_t)b * ws_stride + k] += scale * acc;
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// activation tensor [B,H,W,C] bf16 -> boxes of [1, 16, 16, 64]
static bool make_act_map(CUtensorMap* tm, const __nv_bfloat16* base, int B, int H, int W, int C) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {kKBlock, kTileW, kTileH, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  return encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<__nv_bfloat16*>(base), dims, strides,
                     box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// weights [taps][N][C] bf16 -> boxes of [1, BN, 64]
static bool make_w_map(CUtensorMap* tm, const __nv_bfloat16* base, int taps, int N, int C, int BN) {
  const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)N, (cuuint64_t)taps};
  const cuuint64_t strides[2] = {(cuuint64_t)C * 2, (cuuint64_t)N * C * 2};
  const cuuint32_t box[3] = {kKBlock, (cuuint32_t)BN, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<__nv_bfloat16*>(base), dims, strides,
                     box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int pick_bn(int N) {
  if (N % 128 == 0) return 128;
  if (N <= 128 && N % 16 == 0) return N;  // 96 (ToRGB), 64, 32
  if (N % 64 == 0) return 64;
  return 0;
}

struct Pair {
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
};

#define NFI_SCUDA(expr)                                                              \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess) {                                                        \
      snprintf(err, err_len, "%s failed: %s", #expr, cudaGetErrorString(e__));       \
      return 2;                                                                      \
    }                                                                                \
  } while (0)

static int sm_count() {
  static int n = []() {
    int dev = 0, v = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();
  return n;
}

// One convolution launch.  `in` [map_B (default B),H,W,C] pair, weights [taps9][N][C] pair.
static int launch_conv(ConvArgs& a, Pair in, Pair wt, int w_taps, cudaStream_t st, char* err,
                       size_t err_len, int map_B = 0) {
  if (encode_fn() == nullptr) {
    snprintf(err, err_len, "cuTensorMapEncodeTiled is not available from this driver");
    return 1;
  }
  a.BN = pick_bn(a.N);
  if (a.BN == 0 || a.C % 8 != 0) {  // (TMA: row pitch a multiple of 16 bytes)
    snprintf(err, err_len, "synthesis conv: unsupported channel counts (Cin %d, Cout %d)", a.C, a.N);
    return 1;
  }
  a.n_tiles_n = a.N / a.BN;
  int m_tiles = 0;
  for (int p = 0; p < a.n_phases; ++p) {
    a.ph_ty[p] = (a.ph_DH[p] + kTileH - 1) / kTileH;
    a.ph_tx[p] = (a.ph_DW[p] + kTileW - 1) / kTileW;
    a.ph_tile0[p] = m_tiles;
    m_tiles += a.ph_ty[p] * a.ph_tx[p];
  }
  for (int p = a.n_phases; p <= kMaxPhases; ++p) a.ph_tile0[p] = m_tiles;
  a.ph_tile0[a.n_phases] = m_tiles;
  const int n_tiles = m_tiles * a.B * a.n_tiles_n;
  CUtensorMap tAh, tAl, tWh, tWl;
  if (map_B == 0) map_B = a.B;
  if (!make_act_map(&tAh, in.hi, map_B, a.H, a.W, a.C) || !make_act_map(&tAl, in.lo, map_B, a.H, a.W, a.C) ||
      !make_w_map(&tWh, wt.hi, w_taps, a.N, a.C, a.BN) || !make_w_map(&tWl, wt.lo, w_taps, a.N, a.C, a.BN)) {
    snprintf(err, err_len, "cuTensorMapEncodeTiled failed (B %d H %d W %d C %d N %d)", a.B, a.H, a.W,
             a.C, a.N);
    return 1;
  }
  const int smem = kStages * (2 * kATile + 2 * a.BN * 128) + 128 +
                   ((a.mode == kModeRgb && a.skip != nullptr) ? kSkipBytes : 0);
  NFI_SCUDA(cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  conv_tc_kernel<<<grid, kConvThreads, smem, st>>>(tAh, tAl, tWh, tWl, a, n_tiles);
  NFI_SCUDA(cudaGetLastError());
  return 0;
}

static void conv3x3_phases(ConvArgs& a, int H, int W) {  // stride 1, pad 1 (cross-correlation)
  a.n_phases = 1;
  a.ph_taps[0] = 9;
  a.ph_tap0[0] = 0;
  a.ph_DH[0] = H;
  a.ph_DW[0] = W;
  a.ph_oy[0] = a.ph_ox[0] = 0;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      a.tap_dy[t] = ky - 1;
      a.tap_dx[t] = kx - 1;
      a.tap_w[t] = t;
    }
}
// conv_transpose2d(stride 2): out[2i+ky, 2j+kx] += x[i,j] W[ky,kx].  Output parity (py,px) takes the
// taps with ky = py (mod 2), kx = px (mod 2); position (a,b) of the phase reads x[a - ky/2, b - kx/2].
static void conv_up_phases(ConvArgs& a, int H, int W) {
  a.n_phases = 4;
  int t = 0;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      const int p = py * 2 + px;
      a.ph_tap0[p] = t;
      a.ph_DH[p] = py ? H : H + 1;
      a.ph_DW[p] = px ? W : W + 1;
      a.ph_oy[p] = py;
      a.ph_ox[p] = px;
      for (int ky = py; ky < 3; ky += 2)
        for (int kx = px; kx < 3; kx += 2) {
          a.tap_dy[t] = -(ky / 2);
          a.tap_dx[t] = -(kx / 2);
          a.tap_w[t] = ky * 3 + kx;
          ++t;
        }
      a.ph_taps[p] = t - a.ph_tap0[p];
    }
}

struct Bump {
  unsigned char* base;
  size_t off, cap;
  float* take(size_t floats) {
    const size_t bytes = (floats * sizeof(float) + 1023) & ~(size_t)1023;
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += bytes;
    return p;
  }
  Pair pair(size_t elems) {  // two bf16 tensors of `elems` elements
    Pair p;
    p.hi = reinterpret_cast<__nv_bfloat16*>(take((elems + 1) / 2));
    p.lo = reinterpret_cast<__nv_bfloat16*>(take((elems + 1) / 2));
    return p;
  }
};

static int check_params(const nfi_synth_params& P, char* err, size_t err_len) {
  const int R = P.img_resolution;
  int nb = 0;
  for (int r = 4; r <= R; r <<= 1) ++nb;
  if (R < 8 || (R & (R - 1)) || nb != P.num_blocks || nb > NFI_SYNTH_MAX_BLOCKS) {
    snprintf(err, err_len, "synthesis: img_resolution %d / num_blocks %d inconsistent", R, P.num_blocks);
    return 1;
  }
  if (P.img_channels != 96) {
    snprintf(err, err_len, "synthesis: img_channels must be 96 (3 planes x 32), got %d", P.img_channels);
    return 1;
  }
  if (P.num_ws < 2 * nb) {
    snprintf(err, err_len, "synthesis: ws has %d rows, need %d", P.num_ws, 2 * nb);
    return 1;
  }
  for (int i = 0; i < nb; ++i)
    if (P.channels[i] % 32 != 0 || pick_bn(P.channels[i]) == 0) {
      snprintf(err, err_len, "synthesis: block %d has %d channels (need a multiple of 32 that tiles)", i,
               P.channels[i]);
      return 1;
    }
  return 0;
}

// What the backward reads of a saved forward: pointers into the workspace, recovered by walking the
// same (deterministic) bump allocation again without launching anything.
struct Saved {
  float* style0[NFI_SYNTH_MAX_BLOCKS];
  float* style1[NFI_SYNTH_MAX_BLOCKS];
  float* style_rgb[NFI_SYNTH_MAX_BLOCKS];
  float* dco0[NFI_SYNTH_MAX_BLOCKS];
  float* dco1[NFI_SYNTH_MAX_BLOCKS];
  float* wsq0[NFI_SYNTH_MAX_BLOCKS];
  float* wsq1[NFI_SYNTH_MAX_BLOCKS];
  float* u0[NFI_SYNTH_MAX_BLOCKS];  // pre-activations [B,res,res,cout] (save mode)
  float* u1[NFI_SYNTH_MAX_BLOCKS];
  int row0[NFI_SYNTH_MAX_BLOCKS], row1[NFI_SYNTH_MAX_BLOCKS], row_rgb[NFI_SYNTH_MAX_BLOCKS];
};

// Runs (or, with dry, only lays out) the whole network.  With `sv`, the forward also stores every
// layer's pre-activation u (the save mode) and `sv` receives the pointers the backward reads.
static int run(const nfi_synth_params& P, Bump& ws, cudaStream_t st, bool dry, char* err, size_t err_len,
               Saved* sv = nullptr) {
  const int B = P.batch, nb = P.num_blocks, D = P.w_dim;
  const float sqrt2 = 1.4142135623730951f;
  auto blocks = [](size_t n, int per) { return (unsigned)((n + per - 1) / per); };

  // ---- per-layer styles, demodulation coefficients, re-laid-out weights ----
  float* style0[NFI_SYNTH_MAX_BLOCKS] = {nullptr};
  float* style1[NFI_SYNTH_MAX_BLOCKS] = {nullptr};
  float* style_rgb[NFI_SYNTH_MAX_BLOCKS] = {nullptr};
  float* dco0[NFI_SYNTH_MAX_BLOCKS] = {nullptr};
  float* dco1[NFI_SYNTH_MAX_BLOCKS] = {nullptr};
  Pair w0[NFI_SYNTH_MAX_BLOCKS], w1[NFI_SYNTH_MAX_BLOCKS], wrgb[NFI_SYNTH_MAX_BLOCKS];
  int w_idx = 0;
  for (int i = 0; i < nb; ++i) {
    const int cout = P.channels[i], cin = i ? P.channels[i - 1] : 0;
    const int n_conv = i ? 2 : 1;
    auto style = [&](const nfi_synth_layer& L, int c, int widx, float gain) -> float* {
      float* s = ws.take((size_t)B * c);
      if (!dry)
        styles_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
            P.ws + (size_t)widx * D, P.num_ws * D, D, L.affine_w, L.affine_b, c, B, gain, s);
      return s;
    };
    float* wsq = nullptr;
    auto weights = [&](const nfi_synth_layer& L, int co, int ci, int taps, float* s, Pair& w) -> float* {
      w = ws.pair((size_t)taps * co * ci);
      wsq = taps > 1 ? ws.take((size_t)co * ci) : nullptr;
      float* d = taps > 1 ? ws.take((size_t)B * co) : nullptr;
      if (!dry) {
        prep_weights_kernel<<<blocks((size_t)co * ci, 256), 256, 0, st>>>(L.weight, co, ci, taps, w.hi,
                                                                          w.lo, wsq);
        if (taps > 1)
          dcoef_kernel<<<blocks((size_t)B * co * 32, 256), 256, 0, st>>>(wsq, s, co, ci, B, d);
      }
      return d;
    };
    if (i) {
      style0[i] = style(P.conv0[i], cin, w_idx, 1.f);
      dco0[i] = weights(P.conv0[i], cout, cin, 9, style0[i], w0[i]);
      if (sv) { sv->wsq0[i] = wsq; sv->row0[i] = w_idx; }
    }
    style1[i] = style(P.conv1[i], cout, w_idx + n_conv - 1, 1.f);
    dco1[i] = weights(P.conv1[i], cout, cout, 9, style1[i], w1[i]);
    if (sv) { sv->wsq1[i] = wsq; sv->row1[i] = w_idx + n_conv - 1; }
    // OutputLayer: styles * 1/sqrt(cin * 1 * 1), no demodulation (stylegan.py:369,372-376)
    style_rgb[i] = style(P.torgb[i], cout, w_idx + n_conv, 1.f / sqrtf((float)cout));
    weights(P.torgb[i], P.img_channels, cout, 1, nullptr, wrgb[i]);
    if (sv) sv->row_rgb[i] = w_idx + n_conv;
    w_idx += n_conv;
  }

  if (sv) {
    for (int i = 0; i < nb; ++i) {
      sv->style0[i] = style0[i]; sv->style1[i] = style1[i]; sv->style_rgb[i] = style_rgb[i];
      sv->dco0[i] = dco0[i]; sv->dco1[i] = dco1[i];
      const size_t n = (size_t)B * (4 << i) * (4 << i) * P.channels[i];
      sv->u0[i] = i ? ws.take(n) : nullptr;
      sv->u1[i] = ws.take(n);
    }
  }

  // ---- the blocks ----
  Pair x;                  // input of the next conv (already scaled by its style)
  float* img_prev = nullptr;
  {
    const int C = P.channels[0];
    x = ws.pair((size_t)B * 16 * C);
    if (!dry)
      const_input_kernel<<<blocks((size_t)B * 16 * C, 256), 256, 0, st>>>(P.const_input, style1[0], B, C,
                                                                         x.hi, x.lo);
  }
  for (int i = 0; i < nb; ++i) {
    const int res = 4 << i, cout = P.channels[i], cin = i ? P.channels[i - 1] : cout;
    const bool last = (i == nb - 1);
    if (i) {
      // conv0: transposed conv (4 phase GEMMs over the res/2 grid) -> raw (res+1)^2 -> FIR + ACT
      const int hin = res / 2;
      float* raw = ws.take((size_t)B * (res + 1) * (res + 1) * cout);
      Pair y = ws.pair((size_t)B * res * res * cout);
      if (!dry) {
        ConvArgs a;
        memset(&a, 0, sizeof(a));
        a.B = B; a.C = cin; a.N = cout; a.H = hin; a.W = hin;
        conv_up_phases(a, hin, hin);
        a.mode = kModeRaw;
        a.out_raw = raw; a.out_H = res + 1; a.out_W = res + 1; a.out_stride = 2;
        const int rc = launch_conv(a, x, w0[i], 9, st, err, err_len);
        if (rc) return rc;
        ActEpilogue e;
        memset(&e, 0, sizeof(e));
        e.dcoef = dco0[i]; e.noise = P.conv0[i].noise; e.bias = P.conv0[i].bias; e.gain = sqrt2;
        e.style_a = style1[i]; e.a_hi = y.hi; e.a_lo = y.lo;
        e.u_out = sv ? sv->u0[i] : nullptr;
        const size_t total = (size_t)B * (res / 2) * (res / 2) * (cout / 4);
        unsigned grid = blocks(total, 256);
        if (grid > (unsigned)sm_count() * 16u) grid = (unsigned)sm_count() * 16u;
        fir_act_kernel<<<grid, 256, 0, st>>>(raw, B, res, res, cout, e);
        NFI_SCUDA(cudaGetLastError());
      }
      x = y;
    }
    // conv1 (stride 1) with the fused ACT epilogue; consumers: next block's conv0 and this ToRGB
    Pair xn = {nullptr, nullptr};
    if (!last) xn = ws.pair((size_t)B * res * res * cout);
    Pair xr = ws.pair((size_t)B * res * res * cout);
    if (!dry) {
      ConvArgs a;
      memset(&a, 0, sizeof(a));
      a.B = B; a.C = cout; a.N = cout; a.H = res; a.W = res;
      conv3x3_phases(a, res, res);
      a.mode = kModeAct;
      a.act.dcoef = dco1[i]; a.act.noise = P.conv1[i].noise; a.act.bias = P.conv1[i].bias;
      a.act.gain = sqrt2;
      a.act.style_a = style_rgb[i]; a.act.a_hi = xr.hi; a.act.a_lo = xr.lo;
      if (!last) { a.act.style_b = style0[i + 1]; a.act.b_hi = xn.hi; a.act.b_lo = xn.lo; }
      a.act.u_out = sv ? sv->u1[i] : nullptr;
      const int rc = launch_conv(a, x, w1[i], 9, st, err, err_len);
      if (rc) return rc;
    }
    // ToRGB (1x1, K = cout) + bias + upsampled running image
    float* img = last ? nullptr : ws.take((size_t)B * res * res * P.img_channels);
    if (!dry) {
      ConvArgs a;
      memset(&a, 0, sizeof(a));
      a.B = B; a.C = cout; a.N = P.img_channels; a.H = res; a.W = res;
      a.n_phases = 1; a.ph_taps[0] = 1; a.ph_tap0[0] = 0; a.ph_DH[0] = res; a.ph_DW[0] = res;
      a.tap_dy[0] = a.tap_dx[0] = a.tap_w[0] = 0;
      a.mode = kModeRgb;
      a.act.bias = P.torgb[i].bias;
      a.skip = img_prev; a.img = img; a.planes = last ? P.planes : nullptr;
      const int rc = launch_conv(a, xr, wrgb[i], 1, st, err, err_len);
      if (rc) return rc;
    }
    img_prev = img;
    x = xn;
  }
  return 0;
}

size_t workspace_bytes(const nfi_synth_params& P) {
  Bump b{nullptr, 0, 0};
  char err[256];
  if (check_params(P, err, sizeof(err))) return 0;
  run(P, b, nullptr, true, err, sizeof(err));
  return b.off + 1024;
}

int forward(const nfi_synth_params& P, cudaStream_t st, char* err, size_t err_len) {
  const int rc = check_params(P, err, err_len);
  if (rc) return rc;
  if (P.ws == nullptr || P.const_input == nullptr || P.planes == nullptr || P.workspace == nullptr) {
    snprintf(err, err_len, "synthesis: ws, const_input, planes and workspace must be set");
    return 1;
  }
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need) {
    snprintf(err, err_len, "synthesis: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
    return 1;
  }
  unsigned char* base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(P.workspace) + 1023) & ~(uintptr_t)1023);
  Bump b{base, 0, P.workspace_bytes};
  return run(P, b, st, false, err, err_len);
}

// ---- backward ----
// Walks the blocks from the last to the first.  Scratch reused across blocks (stream order keeps the
// reuse safe): bufA holds g_rgb, then dx~ of conv1, then the raw-gradient phases of conv0; bufB the
// dacc of conv1 (pair), then of conv0 (fp32); bufC dx~ of conv0 until the previous block's conv1
// has consumed it.
static int run_backward(const nfi_synth_params& P, const nfi_synth_grads& G, const Saved& sv, Bump& ws,
                        cudaStream_t st, bool dry, char* err, size_t err_len) {
  const int B = P.batch, nb = P.num_blocks, D = P.w_dim, R = P.img_resolution, NI = P.img_channels;
  const float sqrt2 = 1.4142135623730951f;
  auto blocks = [](size_t n, int per) { return (unsigned)((n + per - 1) / per); };
  auto flat_grid = [&](size_t n) {
    unsigned g = blocks(n, 256);
    return g > (unsigned)sm_count() * 16u ? (unsigned)sm_count() * 16u : g;
  };
  int cmax = 0;
  for (int i = 0; i < nb; ++i) cmax = P.channels[i] > cmax ? P.channels[i] : cmax;
  const size_t full = (size_t)B * R * R * cmax;
  const size_t phases = (size_t)4 * B * (R / 2 + 1) * (R / 2 + 1) * cmax;
  float* bufA = ws.take(full > phases ? full : phases);
  float* bufB = ws.take(full);
  float* bufC = ws.take((size_t)B * (R / 2) * (R / 2) * cmax);
  float* dimg[2] = {ws.take((size_t)B * R * R * NI), ws.take((size_t)B * R * R * NI)};
  Pair dimg_p = ws.pair((size_t)B * R * R * NI);
  // per-(b, channel) sums, zeroed once
  float *ds0[NFI_SYNTH_MAX_BLOCKS], *ds1[NFI_SYNTH_MAX_BLOCKS], *dsr[NFI_SYNTH_MAX_BLOCKS];
  float *dd0[NFI_SYNTH_MAX_BLOCKS], *dd1[NFI_SYNTH_MAX_BLOCKS];
  size_t small = 0;
  for (int i = 0; i < nb; ++i) small += (size_t)B * (4 * P.channels[i] + (i ? P.channels[i - 1] : 0));
  float* sums = ws.take(small);
  {
    float* q = sums;
    for (int i = 0; i < nb; ++i) {
      const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
      ds0[i] = q; q += (size_t)B * ci;
      ds1[i] = q; q += (size_t)B * c;
      dsr[i] = q; q += (size_t)B * c;
      dd0[i] = q; q += (size_t)B * c;
      dd1[i] = q; q += (size_t)B * c;
    }
  }
  Pair wt0[NFI_SYNTH_MAX_BLOCKS], wt1[NFI_SYNTH_MAX_BLOCKS], wtr[NFI_SYNTH_MAX_BLOCKS];
  for (int i = 0; i < nb; ++i) {
    const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
    if (i) wt0[i] = ws.pair((size_t)9 * c * ci);
    wt1[i] = ws.pair((size_t)9 * c * c);
    wtr[i] = ws.pair((size_t)NI * c);
  }
  if (dry) return 0;

  NFI_SCUDA(cudaMemsetAsync(sums, 0, small * sizeof(float), st));
  for (int i = 0; i < nb; ++i) {
    const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
    if (i)
      prep_weights_t_kernel<<<blocks((size_t)c * ci, 256), 256, 0, st>>>(P.conv0[i].weight, c, ci, 9,
                                                                         wt0[i].hi, wt0[i].lo);
    prep_weights_t_kernel<<<blocks((size_t)c * c, 256), 256, 0, st>>>(P.conv1[i].weight, c, c, 9,
                                                                       wt1[i].hi, wt1[i].lo);
    prep_weights_t_kernel<<<blocks((size_t)NI * c, 256), 256, 0, st>>>(P.torgb[i].weight, NI, c, 1,
                                                                       wtr[i].hi, wtr[i].lo);
  }
  planes_grad_kernel<<<flat_grid((size_t)B * R * R * NI), 256, 0, st>>>(G.g_planes, B, R, dimg[0],
                                                                        dimg_p.hi, dimg_p.lo);
  NFI_SCUDA(cudaGetLastError());

  auto act_backward = [&](ActBackward& e, int HW, int C) -> int {
    if (C % 4 != 0 || C / 4 > 256) {
      snprintf(err, err_len, "synthesis backward: %d channels unsupported", C);
      return 1;
    }
    const int chunk = 1024;
    dim3 grid((unsigned)((HW + chunk - 1) / chunk), (unsigned)B);
    act_backward_kernel<<<grid, 256, 0, st>>>(e, HW, C, chunk);
    NFI_SCUDA(cudaGetLastError());
    return 0;
  };
  auto to_ws = [&](const float* ds, const nfi_synth_layer& L, int cin, int row, float gain) {
    styles_backward_kernel<<<blocks((size_t)B * D, 256), 256, 0, st>>>(
        ds, L.affine_w, cin, D, B, gain / sqrtf((float)D), G.g_ws + (size_t)row * D, P.num_ws * D);
  };
  auto stride1_taps = [](ConvArgs& a, int H, int W) {  // the adjoint of conv3x3_phases: taps flipped
    conv3x3_phases(a, H, W);
    for (int t = 0; t < 9; ++t) {
      a.tap_dy[t] = -a.tap_dy[t];
      a.tap_dx[t] = -a.tap_dx[t];
    }
  };

  int cur = 0;  // dimg[cur] is the gradient of block i's running image
  for (int i = nb - 1; i >= 0; --i) {
    const int res = 4 << i, c = P.channels[i], ci = i ? P.channels[i - 1] : 0, HW = res * res;
    const bool last = (i == nb - 1);
    // ToRGB: g = dimg Wrgb^T  [B,res,res,c] -> bufA
    {
      ConvArgs a;
      memset(&a, 0, sizeof(a));
      a.B = B; a.C = NI; a.N = c; a.H = res; a.W = res;
      a.n_phases = 1; a.ph_taps[0] = 1; a.ph_DH[0] = res; a.ph_DW[0] = res;
      a.mode = kModeRaw;
      a.out_raw = bufA; a.out_H = res; a.out_W = res; a.out_stride = 1;
      const int rc = launch_conv(a, dimg_p, wtr[i], 1, st, err, err_len);
      if (rc) return rc;
    }
    if (i) {  // the running image's gradient one block down (the GEMM above has read dimg_p)
      const int h = res / 2;
      upsample_adjoint_kernel<<<flat_grid((size_t)B * h * h * NI), 256, 0, st>>>(
          dimg[cur], B, h, h, NI, dimg[cur ^ 1], dimg_p.hi, dimg_p.lo);
      NFI_SCUDA(cudaGetLastError());
      cur ^= 1;
    }
    // conv1: consumers ToRGB (style_rgb) and, below the last block, conv0 of block i+1 (bufC)
    {
      ActBackward e;
      memset(&e, 0, sizeof(e));
      e.u = sv.u1[i]; e.noise = P.conv1[i].noise; e.bias = P.conv1[i].bias; e.dcoef = sv.dco1[i];
      e.gain = sqrt2;
      e.dx_a = bufA; e.s_a = sv.style_rgb[i]; e.ds_a = dsr[i];
      if (!last) { e.dx_b = bufC; e.s_b = sv.style0[i + 1]; e.ds_b = ds0[i + 1]; }
      e.dd = dd1[i];
      Pair pb = {reinterpret_cast<__nv_bfloat16*>(bufB),
                 reinterpret_cast<__nv_bfloat16*>(bufB) + (size_t)B * HW * c};
      e.dacc_hi = pb.hi; e.dacc_lo = pb.lo;
      if (int rc = act_backward(e, HW, c)) return rc;
      to_ws(dsr[i], P.torgb[i], c, sv.row_rgb[i], 1.f / sqrtf((float)c));
      if (!last) {
        const int cn = P.channels[i + 1];
        dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
            sv.wsq0[i + 1], sv.style0[i + 1], dd0[i + 1], sv.dco0[i + 1], cn, c, B, ds0[i + 1]);
        to_ws(ds0[i + 1], P.conv0[i + 1], c, sv.row0[i + 1], 1.f);
      }
      // dx~ of conv1 = conv^T(dacc, W1) -> bufA
      ConvArgs a;
      memset(&a, 0, sizeof(a));
      a.B = B; a.C = c; a.N = c; a.H = res; a.W = res;
      stride1_taps(a, res, res);
      a.mode = kModeRaw;
      a.out_raw = bufA; a.out_H = res; a.out_W = res; a.out_stride = 1;
      const int rc = launch_conv(a, pb, wt1[i], 9, st, err, err_len);
      if (rc) return rc;
    }
    if (i == 0) {
      const_ds_kernel<<<blocks((size_t)B * c, 256), 256, 0, st>>>(bufA, P.const_input, B, c, ds1[0]);
      dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
          sv.wsq1[0], sv.style1[0], dd1[0], sv.dco1[0], c, c, B, ds1[0]);
      to_ws(ds1[0], P.conv1[0], c, sv.row1[0], 1.f);
      NFI_SCUDA(cudaGetLastError());
      break;
    }
    // conv0 (up): its one consumer is conv1 -> dacc fp32 in bufB, ds1 and dd0
    {
      ActBackward e;
      memset(&e, 0, sizeof(e));
      e.u = sv.u0[i]; e.noise = P.conv0[i].noise; e.bias = P.conv0[i].bias; e.dcoef = sv.dco0[i];
      e.gain = sqrt2;
      e.dx_a = bufA; e.s_a = sv.style1[i]; e.ds_a = ds1[i];
      e.dd = dd0[i];
      e.dacc = bufB;
      if (int rc = act_backward(e, HW, c)) return rc;
      dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
          sv.wsq1[i], sv.style1[i], dd1[i], sv.dco1[i], c, c, B, ds1[i]);
      to_ws(ds1[i], P.conv1[i], c, sv.row1[i], 1.f);
    }
    // FIR adjoint -> the four parity phases of the raw gradient (pair in bufA), then the
    // stride-2 correlation with W0 as 9 stride-1 taps over them -> dx~ of conv0 in bufC
    {
      const int h = res / 2;
      Pair ph = {reinterpret_cast<__nv_bfloat16*>(bufA),
                 reinterpret_cast<__nv_bfloat16*>(bufA) + (size_t)4 * B * (h + 1) * (h + 1) * c};
      fir_adjoint_kernel<<<flat_grid((size_t)4 * B * (h + 1) * (h + 1) * (c / 4)), 256, 0, st>>>(
          bufB, B, res, res, c, ph.hi, ph.lo);
      NFI_SCUDA(cudaGetLastError());
      ConvArgs a;
      memset(&a, 0, sizeof(a));
      a.B = B; a.C = c; a.N = ci; a.H = h + 1; a.W = h + 1;
      a.n_phases = 1; a.ph_taps[0] = 9; a.ph_DH[0] = h; a.ph_DW[0] = h;
      for (int ky = 0; ky < 3; ++ky)
        for (int kx = 0; kx < 3; ++kx) {
          const int t = ky * 3 + kx;
          a.tap_dy[t] = ky / 2;
          a.tap_dx[t] = kx / 2;
          a.tap_w[t] = t;
          a.tap_img[t] = ((ky & 1) * 2 + (kx & 1)) * B;
        }
      a.mode = kModeRaw;
      a.out_raw = bufC; a.out_H = h; a.out_W = h; a.out_stride = 1;
      const int rc = launch_conv(a, ph, wt0[i], 9, st, err, err_len, 4 * B);
      if (rc) return rc;
    }
  }
  NFI_SCUDA(cudaGetLastError());
  return 0;
}

static int saved_layout(const nfi_synth_params& P, Bump& b, Saved& sv, char* err, size_t err_len) {
  return run(P, b, nullptr, true, err, err_len, &sv);
}

size_t saved_workspace_bytes(const nfi_synth_params& P) {
  char err[256];
  if (check_params(P, err, sizeof(err))) return 0;
  Bump b{nullptr, 0, 0};
  Saved sv;
  memset(&sv, 0, sizeof(sv));
  saved_layout(P, b, sv, err, sizeof(err));
  nfi_synth_grads g = {nullptr, nullptr};
  run_backward(P, g, sv, b, nullptr, true, err, sizeof(err));
  return b.off + 1024;
}

static int check_saved(const nfi_synth_params& P, char* err, size_t err_len) {
  const int rc = check_params(P, err, err_len);
  if (rc) return rc;
  if (P.ws == nullptr || P.const_input == nullptr || P.planes == nullptr || P.workspace == nullptr) {
    snprintf(err, err_len, "synthesis: ws, const_input, planes and workspace must be set");
    return 1;
  }
  const size_t need = saved_workspace_bytes(P);
  if (P.workspace_bytes < need) {
    snprintf(err, err_len, "synthesis: saved workspace too small (%zu < %zu bytes)", P.workspace_bytes,
             need);
    return 1;
  }
  return 0;
}

int forward_saved(const nfi_synth_params& P, cudaStream_t st, char* err, size_t err_len) {
  if (const int rc = check_saved(P, err, err_len)) return rc;
  unsigned char* base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(P.workspace) + 1023) & ~(uintptr_t)1023);
  Bump b{base, 0, P.workspace_bytes};
  Saved sv;
  memset(&sv, 0, sizeof(sv));
  return run(P, b, st, false, err, err_len, &sv);
}

int backward(const nfi_synth_params& P, const nfi_synth_grads& G, cudaStream_t st, char* err,
             size_t err_len) {
  if (const int rc = check_saved(P, err, err_len)) return rc;
  if (G.g_planes == nullptr || G.g_ws == nullptr) {
    snprintf(err, err_len, "synthesis backward: g_planes and g_ws must be set");
    return 1;
  }
  unsigned char* base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(P.workspace) + 1023) & ~(uintptr_t)1023);
  Bump b{base, 0, P.workspace_bytes};
  Saved sv;
  memset(&sv, 0, sizeof(sv));
  if (const int rc = saved_layout(P, b, sv, err, err_len)) return rc;
  return run_backward(P, G, sv, b, st, false, err, err_len);
}

}  // namespace synth
}  // namespace nfi
