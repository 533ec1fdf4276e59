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
#include <string.h>

#include "nfi_pair.cuh"
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
  const float* dcoef;  // [B,N] or nullptr (1: no demodulation, the LPIPS network's plain convs)
  const float* noise;  // [B,H,W] or nullptr
  const float* bias;   // [N]
  float gain;          // sqrt(2)
  float slope;         // negative slope of the activation: 0.2 (leaky ReLU), 0 (ReLU)
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

constexpr float kSlope = 0.2f;  // the leaky ReLU's negative slope

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
  const float2 d = e.dcoef ? __ldg(reinterpret_cast<const float2*>(e.dcoef + (size_t)img * N + n))
                          : make_float2(1.f, 1.f);
  const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + n));
  float2 u, v;
  u.x = ((acc.x * d.x + noise) + b.x) * e.gain;
  u.y = ((acc.y * d.y + noise) + b.y) * e.gain;
  if (e.u_out != nullptr) *reinterpret_cast<float2*>(e.u_out + pos * N + n) = u;
  v.x = lrelu(u.x, e.slope);
  v.y = lrelu(u.y, e.slope);
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
  const float4 d = e.dcoef ? __ldg(reinterpret_cast<const float4*>(e.dcoef + (size_t)img * N + n))
                          : make_float4(1.f, 1.f, 1.f, 1.f);
  const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + n));
  float4 u, v;
  u.x = ((acc.x * d.x + noise) + b.x) * e.gain;
  u.y = ((acc.y * d.y + noise) + b.y) * e.gain;
  u.z = ((acc.z * d.z + noise) + b.z) * e.gain;
  u.w = ((acc.w * d.w + noise) + b.w) * e.gain;
  if (e.u_out != nullptr) *reinterpret_cast<float4*>(e.u_out + pos * N + n) = u;
  v.x = lrelu(u.x, e.slope);
  v.y = lrelu(u.y, e.slope);
  v.z = lrelu(u.z, e.slope);
  v.w = lrelu(u.w, e.slope);
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

// The tangent of the ACT epilogue along ws (the path-length HVP's forward pass): with acc-dot the
// conv of the tangent input, u-dot = gain (acc-dot d + acc d-dot), acc d = u / gain - noise - bias
// recovered from the saved u (noise and bias do not depend on ws).
struct TangentEpilogue {
  const float* dcoef;  // [B,N] d
  const float* ddot;   // [B,N] d-dot
  const float* noise;  // [B,H,W] or nullptr
  const float* bias;   // [N]
  const float* u;      // [B,H,W,N] saved pre-activation
  float gain;
  float* u_dot;        // [B,H,W,N] out
};
__device__ __forceinline__ void act_store4(const TangentEpilogue& e, int img, size_t pos, int N, int n,
                                           float4 acc, float noise) {
  const float4 d = __ldg(reinterpret_cast<const float4*>(e.dcoef + (size_t)img * N + n));
  const float4 dd = __ldg(reinterpret_cast<const float4*>(e.ddot + (size_t)img * N + n));
  const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + n));
  const float4 u = __ldg(reinterpret_cast<const float4*>(e.u + pos * N + n));
  const float ig = 1.f / e.gain;
  float4 o;
  o.x = (acc.x * d.x + (u.x * ig - noise - b.x) * (dd.x / d.x)) * e.gain;
  o.y = (acc.y * d.y + (u.y * ig - noise - b.y) * (dd.y / d.y)) * e.gain;
  o.z = (acc.z * d.z + (u.z * ig - noise - b.z) * (dd.z / d.z)) * e.gain;
  o.w = (acc.w * d.w + (u.w * ig - noise - b.w) * (dd.w / d.w)) * e.gain;
  *reinterpret_cast<float4*>(e.u_dot + pos * N + n) = o;
}

// 4x4 FIR (outer([1,3,3,1]) / 16 = the reference's filter * gain 4, pad 1) over the (2H+1)x(2W+1)
// transposed-conv result, then the ACT epilogue (or its tangent).  One thread per (2x2 output
// block, 4 channels): the block needs a 5x5 window of the raw tensor (25 loads for 4 outputs
// instead of 16 each), rows filtered first (separable), then columns.
template <class Epilogue>
__global__ void __launch_bounds__(256)
fir_act_kernel(const float* __restrict__ raw, int B, int OH, int OW, int N, Epilogue e) {
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

// The forward's weight prep: weight [Cout,Cin,K,K] -> [K*K][Cout][Cin] hi / lo (K-major rows of the
// B operand) and wsq[Cout][Cin] = sum over taps of W^2 (for the demodulation coefficients)
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
// 329,372); one warp per (b, c).  affine_b NULL: the style's tangent along w (no bias term).
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
  if (lane == 0) out[warp] = (s * rsqrtf((float)w_dim) + (ab ? ab[c] : 0.f)) * gain;
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
// re-laid-out by prep_weights (kTapCiCo: the B operand of a GEMM that reduces over Cout; the
// stride-1 layer's tap flip lives in the tap table); everything between two GEMMs of a layer is
// ONE full-resolution pass (act_backward_kernel), plus the FIR adjoint for the up layers.

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
  // parameter backward only (act_backward_kernel<true>): += sum_{b,pos} g and += sum_c g
  float* g_bias;           // [C]
  float* g_noise;          // [B,HW] (with noise)
};

constexpr int kActChunk = 1024;  // positions per block of act_backward_kernel

// One pass over a layer's output: dv = dx~_a s_a + dx~_b s_b, then dacc = dv lrelu'(u) gain d, and
// the per-(b, channel) sums ds_a, ds_b, dd.  Block (chunk, b): 4 channels per thread, 256 / (C/4)
// positions in parallel; the sums are reduced in shared memory, then one atomic per block.
// kParams adds the bias sum of g (a fourth per-block reduction) and the noise gradient sum_c g per
// position (shared atomics over the block's chunk, then one plain += per position: each position
// belongs to one block); every other value is computed as without it.
template <bool kParams>
__global__ void __launch_bounds__(256)
act_backward_kernel(ActBackward e, int HW, int C, int chunk) {
  __shared__ float4 red[kParams ? 4 : 3][256];
  __shared__ float nsum[kParams ? kActChunk : 1];
  if constexpr (kParams) {
    for (int i = threadIdx.x; i < kActChunk; i += 256) nsum[i] = 0.f;
    __syncthreads();
  }
  float4 sg = make_float4(0.f, 0.f, 0.f, 0.f);
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
    acc.x = fmaf(x.x, lrelu(u.x, kSlope), acc.x);                                   \
    acc.y = fmaf(x.y, lrelu(u.y, kSlope), acc.y);                                   \
    acc.z = fmaf(x.z, lrelu(u.z, kSlope), acc.z);                                   \
    acc.w = fmaf(x.w, lrelu(u.w, kSlope), acc.w);                                   \
    dv.x = fmaf(x.x, s.x, dv.x); dv.y = fmaf(x.y, s.y, dv.y);                       \
    dv.z = fmaf(x.z, s.z, dv.z); dv.w = fmaf(x.w, s.w, dv.w);                       \
  }
      NFI_CONSUMER(e.dx_a, s_a, sa)
      NFI_CONSUMER(e.dx_b, s_b, sb)
#undef NFI_CONSUMER
      float4 g, out;
#define NFI_G(cmp)                                                                   \
  g.cmp = dv.cmp * lrelu_grad(u.cmp, kSlope) * e.gain;                               \
  sd.cmp = fmaf(g.cmp, u.cmp * inv_gain - nz - bi.cmp, sd.cmp);  /* acc d = u/gain - noise - bias */ \
  out.cmp = g.cmp * d.cmp;
      NFI_G(x) NFI_G(y) NFI_G(z) NFI_G(w)
#undef NFI_G
      if (e.dacc_hi != nullptr) store_split4(e.dacc_hi, e.dacc_lo, idx, out, one);
      if (e.dacc != nullptr) *reinterpret_cast<float4*>(e.dacc + idx) = out;
      if constexpr (kParams) {
        sg.x += g.x; sg.y += g.y; sg.z += g.z; sg.w += g.w;
        if (e.g_noise != nullptr) atomicAdd(&nsum[pos - blockIdx.x * chunk], (g.x + g.y) + (g.z + g.w));
      }
    }
  }
  red[0][tid] = sa;
  red[1][tid] = sb;
  red[2][tid] = sd;
  if constexpr (kParams) red[3][tid] = sg;
  __syncthreads();
  if constexpr (kParams) {
    if (e.g_noise != nullptr) {
      const int p0 = blockIdx.x * chunk, n = min(HW, p0 + chunk) - p0;
      for (int i = tid; i < n; i += 256) e.g_noise[(size_t)b * HW + p0 + i] += nsum[i];
    }
    if (e.g_bias != nullptr && tid < cg) {
      float4 s = red[3][tid];
      for (int k = 1; k < ppar; ++k) {
        const float4 t = red[3][k * cg + tid];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      atomicAdd(e.g_bias + 4 * tid + 0, s.x);
      atomicAdd(e.g_bias + 4 * tid + 1, s.y);
      atomicAdd(e.g_bias + 4 * tid + 2, s.z);
      atomicAdd(e.g_bias + 4 * tid + 3, s.w);
    }
  }
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

// ------------------------------------------------------------------ backward to the parameters
// dW[co,ci,tap] = sum_{b,p} G_b[p + a_off(tap), co] X_b[p + x_off(tap), ci]: G is the gradient of
// the conv output before demodulation (dacc, the up layer's four raw-gradient phases, or dimg for
// ToRGB) and X the layer's styled input x~, both position-major [B,H,W,C] bf16 pairs.  A k-tile is
// 16 x 4 positions: one [64 ch x 64 positions] TMA box per operand (128-byte rows, SWIZZLE_128B),
// which is the MN-major wgmma operand as it lands (K = positions; out-of-range rows / columns /
// channels arrive as zeros = the 3x3 padding).  A work item is (Cout tile, Cin tile, tap, K range);
// it runs its K range as chains of kWgChain k-tiles (A_lo X_hi + A_hi X_lo + A_hi X_hi, fp32
// accumulate in registers), adds each chain into an fp32 total in registers, and stores the total
// to its own slice of a partials buffer; wgrad_reduce_kernel sums the slices in a fixed order.
//
// wgrad_tc_kernel (persistent, 160 threads, two CTAs per SM):
//   warps 0-3   consumer warpgroup: D[64 co x 64 ci], 12 wgmma (bf16, M64 N64 K16) per k-tile
//   warp 4      TMA producer: 4 boxes per k-tile (G_hi, G_lo, X_hi, X_lo, 8 KB each), 3-stage ring
constexpr int kWgTileH = 4, kWgTileW = 16;
constexpr int kWgBox = 64 * 128;
constexpr int kWgStage = 4 * kWgBox;
constexpr int kWgStages = 3;
constexpr int kWgThreads = 160;
constexpr int kWgChain = 8;          // k-tiles (512 positions) per tensor-core accumulation chain
constexpr int kWgItems = 1024;       // the K split aims at this many work items (device-independent)
constexpr int kWgMinSplit = 16;      // k-tiles per work item at least

struct WgradArgs {
  int kt_y, kt_x, kt_img, kt_total;    // k-tiles per column / row of the domain, per image, all
  int taps;
  int a_dy[kMaxTaps], a_dx[kMaxTaps], a_img[kMaxTaps];  // G box offset of the tap
  int x_dy[kMaxTaps], x_dx[kMaxTaps];                   // X box offset of the tap
  int cout, cin, n_co, n_ci;           // channels and 64-channel tiles
  int n_split, split_len;              // K ranges of split_len k-tiles
  int chain;                           // k-tiles per chain
  float* part;                         // [n_split][taps][cout][cin]
};

__global__ void __launch_bounds__(kWgThreads, 2)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmGh, const __grid_constant__ CUtensorMap tmGl,
                const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl,
                const __grid_constant__ WgradArgs a, int n_items) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStage);
  uint64_t* empty = full + kWgStages;
  if (tid == 0) {
    if (tc::smem_u32(smem) & 1023u) __trap();
    for (int i = 0; i < kWgStages; ++i) {
      tc::mbar_init(&full[i], 1);
      tc::mbar_init(&empty[i], 4);
    }
    tc::fence_mbar_init();
    prefetch_tmap(&tmGh);
    prefetch_tmap(&tmGl);
    prefetch_tmap(&tmXh);
    prefetch_tmap(&tmXl);
  }
  __syncthreads();
  // item = ((split * taps + tap) * n_co + co) * n_ci + ci: concurrent CTAs share a K range (L2)
  auto decode = [&](int item, int& ci, int& co, int& tap, int& k0, int& k1) {
    ci = item % a.n_ci;
    int r = item / a.n_ci;
    co = r % a.n_co;
    r /= a.n_co;
    tap = r % a.taps;
    const int split = r / a.taps;
    k0 = split * a.split_len;
    k1 = min(a.kt_total, k0 + a.split_len);
  };

  if (__shfl_sync(0xffffffffu, tid >> 7, 0) != 0) {
    // ================================ TMA PRODUCER ================================
    if (elect_one()) {
      uint32_t st = 0, ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        int ci, co, tap, k0, k1;
        decode(item, ci, co, tap, k0, k1);
        for (int kt = k0; kt < k1; ++kt) {
          const int img = kt / a.kt_img, r = kt - img * a.kt_img;
          const int ty = r / a.kt_x, tx = r - ty * a.kt_x;
          const int y0 = ty * kWgTileH, x0 = tx * kWgTileW;
          tc::mbar_wait(&empty[st], ph ^ 1);
          unsigned char* s = smem + st * kWgStage;
          tc::mbar_expect_tx(&full[st], (uint32_t)kWgStage);
          tma_load_4d(s, &tmGh, co * 64, x0 + a.a_dx[tap], y0 + a.a_dy[tap], img + a.a_img[tap], &full[st]);
          tma_load_4d(s + kWgBox, &tmGl, co * 64, x0 + a.a_dx[tap], y0 + a.a_dy[tap], img + a.a_img[tap],
                      &full[st]);
          tma_load_4d(s + 2 * kWgBox, &tmXh, ci * 64, x0 + a.x_dx[tap], y0 + a.x_dy[tap], img, &full[st]);
          tma_load_4d(s + 3 * kWgBox, &tmXl, ci * 64, x0 + a.x_dx[tap], y0 + a.x_dy[tap], img, &full[st]);
          if (++st == kWgStages) { st = 0; ph ^= 1; }
        }
      }
    }
    return;
  }
  // ================================ CONSUMER WARPGROUP ================================
  const int lane = tid & 31, warp = tid >> 5;
  const int g4 = lane >> 2, t = lane & 3;
  const uint32_t smem_s = tc::smem_u32(smem);
  uint32_t st = 0, ph = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    int ci, co, tap, k0, k1;
    decode(item, ci, co, tap, k0, k1);
    float tot[32], acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) tot[i] = 0.f;
    for (int c0 = k0; c0 < k1; c0 += a.chain) {
      const int c1 = min(k1, c0 + a.chain);
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      tc::wgmma_fence();
      uint32_t prev_st = 0;
      for (int k = c0; k < c1; ++k) {
        tc::mbar_wait(&full[st], ph);
        const uint32_t sb = smem_s + st * kWgStage;
        // small terms first; a K step of 16 positions = 16 rows of 128 B = 2048 B (two 8-row groups)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          tc::wgmma_bf16_ss_n64<1, 1>(acc, tc::gmma_desc(sb + kWgBox + 2048 * ks, tc::kSw128, 16, 1024),
                                      tc::gmma_desc(sb + 2 * kWgBox + 2048 * ks, tc::kSw128, 16, 1024), 1);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          tc::wgmma_bf16_ss_n64<1, 1>(acc, tc::gmma_desc(sb + 2048 * ks, tc::kSw128, 16, 1024),
                                      tc::gmma_desc(sb + 3 * kWgBox + 2048 * ks, tc::kSw128, 16, 1024), 1);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          tc::wgmma_bf16_ss_n64<1, 1>(acc, tc::gmma_desc(sb + 2048 * ks, tc::kSw128, 16, 1024),
                                      tc::gmma_desc(sb + 2 * kWgBox + 2048 * ks, tc::kSw128, 16, 1024), 1);
        tc::wgmma_commit();
        // the previous stage's products are complete once at most this one's are in flight
        tc::wgmma_wait<1>();
        if (k > c0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev_st]);
        }
        prev_st = st;
        if (++st == kWgStages) { st = 0; ph ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::reg_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev_st]);
#pragma unroll
      for (int i = 0; i < 32; ++i) tot[i] += acc[i];
    }
    // rows co*64 + 16 warp + g4 (+8), columns ci*64 + 8j + 2t (+1)
    const int split = k0 / a.split_len;
    float* dst = a.part + ((size_t)split * a.taps + tap) * a.cout * a.cin;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int o = co * 64 + 16 * warp + g4 + 8 * half;
      if (o >= a.cout) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i = ci * 64 + 8 * j + 2 * t;
        if (i < a.cin) dst[(size_t)o * a.cin + i] = tot[4 * j + 2 * half];
        if (i + 1 < a.cin) dst[(size_t)o * a.cin + i + 1] = tot[4 * j + 2 * half + 1];
      }
    }
  }
}

// g_weight[co,ci,tap] += sum_split part[split][tap][co][ci] (split order fixed) and, for the
// modulated 3x3 layers, the demodulation term: d = rsqrt(sum_ci s^2 sum_taps W^2 + 1e-8) gives
// dd/dW[co,ci,tap] = -d^3 s_ci^2 W, and dd_true = dd_part / d (act_backward_kernel sums g (acc d)),
// so dW -= W sum_b dd_part[b,co] d[b,co]^2 s[b,ci]^2.  One thread per (co, ci).
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int n_split, int taps, int cout,
                                    int cin, const float* __restrict__ w, const float* __restrict__ dd,
                                    const float* __restrict__ d, const float* __restrict__ s, int B,
                                    float* __restrict__ g_w) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)cout * cin;
  if (i >= n) return;
  const int o = (int)(i / cin), c = (int)(i % cin);
  float dem = 0.f;
  if (dd != nullptr)
    for (int b = 0; b < B; ++b) {
      const float dv = d[(size_t)b * cout + o], sv = s[(size_t)b * cin + c];
      dem = fmaf(dd[(size_t)b * cout + o] * dv * dv, sv * sv, dem);
    }
  for (int tp = 0; tp < taps; ++tp) {
    float acc = 0.f;
    for (int sp = 0; sp < n_split; ++sp) acc += part[((size_t)sp * taps + tp) * n + i];
    g_w[i * taps + tp] += acc - w[i * taps + tp] * dem;
  }
}

// x~ = lrelu(u) s as a pair: the same arithmetic as act_store4, so the same bits the forward fed
// the layer's GEMM
__global__ void restyle_kernel(const float* __restrict__ u, const float* __restrict__ s, int B, int HW,
                               int C, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int groups = C >> 2;
  const size_t total = (size_t)B * HW * groups;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int img = (int)(i / ((size_t)HW * groups));
    float4 v = __ldg(reinterpret_cast<const float4*>(u) + i);
    v.x = lrelu(v.x, kSlope); v.y = lrelu(v.y, kSlope);
    v.z = lrelu(v.z, kSlope); v.w = lrelu(v.w, kSlope);
    const float4 sv = __ldg(reinterpret_cast<const float4*>(s + (size_t)img * C) + g);
    store_split4(hi, lo, i * 4, v, sv);
  }
}

// out[c] += sum over rows of x[row, c] (ToRGB bias: sum_{b,p} dimg).  Block: a chunk of rows,
// 256 / C rows in parallel, reduced in shared memory, one atomic per column per block.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ x, size_t rows, int C, int chunk, float* __restrict__ out) {
  __shared__ float red[256];
  const int par = 256 / C, tid = threadIdx.x, r0 = tid / C, c = tid - r0 * C;
  float acc = 0.f;
  if (r0 < par) {
    const size_t end = min(rows, (size_t)(blockIdx.x + 1) * chunk);
    for (size_t r = (size_t)blockIdx.x * chunk + r0; r < end; r += par) acc += x[r * C + c];
  }
  red[tid] = acc;
  __syncthreads();
  if (tid < C) {
    for (int k = 1; k < par; ++k) acc += red[k * C + tid];
    atomicAdd(out + tid, acc);
  }
}

// The affine's gradients from the style gradient ds [B,cin] (styles_kernel's transpose in the
// other operand): g_aw[c,k] += scale sum_b ds[b,c] ws[b,row,k], g_ab[c] += gain sum_b ds[b,c]
__global__ void affine_backward_kernel(const float* __restrict__ ds, const float* __restrict__ ws,
                                       int ws_stride, int B, int cin, int w_dim, float scale, float gain,
                                       float* __restrict__ g_aw, float* __restrict__ g_ab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cin * w_dim) return;
  const int c = i / w_dim, k = i % w_dim;
  float acc = 0.f, sb = 0.f;
  for (int b = 0; b < B; ++b) {
    const float v = ds[(size_t)b * cin + c];
    acc = fmaf(v, ws[(size_t)b * ws_stride + k], acc);
    sb += v;
  }
  if (g_aw != nullptr) g_aw[i] += scale * acc;
  if (g_ab != nullptr && k == 0) g_ab[c] += gain * sb;
}

// b4.const: x~[b,p,c] = const[c,p] s[b,c], so g_const[c,p] += sum_b dx~[b,p,c] s[b,c]
__global__ void const_grad_kernel(const float* __restrict__ dx, const float* __restrict__ s, int B, int C,
                                  float* __restrict__ g_const) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * 16) return;
  const int c = i / 16, p = i % 16;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc = fmaf(dx[((size_t)b * 16 + p) * C + c], s[(size_t)b * C + c], acc);
  g_const[i] += acc;
}

// ------------------------------------------------------------------ path-length HVP
// The gradient of <t, J_ws^T n> with respect to ws and every parameter is the tangent, along
// ws + eps t, of the backward with the planes cotangent n (symmetry of second derivatives).  Every
// backward quantity q gets a tangent q-dot: a tangent forward pass first (s-dot, d-dot, and u-dot
// per layer kept in fp32), then the backward walk recomputed beside its tangent; each GEMM is one
// the backward already runs, on 2B stacked images where a product and its tangent share an operand.

// d-dot[b,o] = -d^3 sum_c wsq[o,c] s s-dot (the tangent of dcoef_kernel); one warp per (b, o)
__global__ void dcoef_tangent_kernel(const float* __restrict__ wsq, const float* __restrict__ s,
                                     const float* __restrict__ sdot, const float* __restrict__ d, int cout,
                                     int cin, int B, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * cout) return;
  const int b = warp / cout, o = warp % cout;
  float acc = 0.f;
  for (int c = lane; c < cin; c += 32)
    acc = fmaf(wsq[(size_t)o * cin + c], s[(size_t)b * cin + c] * sdot[(size_t)b * cin + c], acc);
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, k);
  if (lane == 0) {
    const float dv = d[warp];
    out[warp] = -(dv * dv * dv) * acc;
  }
}

// The tangent ACT pass of a stride-1 layer: acc-dot [B,HW,C] (the RAW conv of the tangent input)
// -> u-dot, through the same epilogue as fir_act_kernel<TangentEpilogue>
__global__ void tangent_act_kernel(const float* __restrict__ acc_dot, int B, int HW, int C, TangentEpilogue e) {
  const int groups = C >> 2;
  const size_t total = (size_t)B * HW * groups;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const size_t pos = i / groups;
    const float noise = e.noise ? __ldg(e.noise + pos) : 0.f;
    act_store4(e, (int)(pos / HW), pos, C, 4 * g, __ldg(reinterpret_cast<const float4*>(acc_dot) + i), noise);
  }
}

// x~-dot = lrelu'(u) u-dot s + lrelu(u) s-dot as a pair: the tangent of restyle_kernel
__global__ void restyle_tangent_kernel(const float* __restrict__ u, const float* __restrict__ udot,
                                       const float* __restrict__ s, const float* __restrict__ sdot, int B,
                                       int HW, int C, __nv_bfloat16* __restrict__ hi,
                                       __nv_bfloat16* __restrict__ lo) {
  const int groups = C >> 2;
  const size_t total = (size_t)B * HW * groups;
  const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int img = (int)(i / ((size_t)HW * groups));
    const float4 v = __ldg(reinterpret_cast<const float4*>(u) + i);
    const float4 vd = __ldg(reinterpret_cast<const float4*>(udot) + i);
    const float4 sv = __ldg(reinterpret_cast<const float4*>(s + (size_t)img * C) + g);
    const float4 sd = __ldg(reinterpret_cast<const float4*>(sdot + (size_t)img * C) + g);
    float4 x;
    x.x = lrelu_grad(v.x, kSlope) * vd.x * sv.x + lrelu(v.x, kSlope) * sd.x;
    x.y = lrelu_grad(v.y, kSlope) * vd.y * sv.y + lrelu(v.y, kSlope) * sd.y;
    x.z = lrelu_grad(v.z, kSlope) * vd.z * sv.z + lrelu(v.z, kSlope) * sd.z;
    x.w = lrelu_grad(v.w, kSlope) * vd.w * sv.w + lrelu(v.w, kSlope) * sd.w;
    store_split4(hi, lo, i * 4, x, one);
  }
}

struct ActBackwardTangent {
  const float* u;       // [B,HW,C] saved pre-activation
  const float* u_dot;   // [B,HW,C] its tangent
  const float* noise;   // [B,HW] or nullptr
  const float* bias;    // [C]
  const float* dcoef;   // [B,C] d
  const float* ddot;    // [B,C] d-dot
  float gain;           // sqrt(2)
  // up to two consumers of v: dx~ and its tangent (nullptr = 0), style and its tangent, and
  // ds += sum_pos dx~ v, ds-dot += sum_pos dx~-dot v + dx~ v-dot
  const float* dx_a; const float* dxt_a; const float* s_a; const float* st_a; float* ds_a; float* dst_a;
  const float* dx_b; const float* dxt_b; const float* s_b; const float* st_b; float* ds_b; float* dst_b;
  float* dd;            // [B,C] += sum_pos g (acc d)
  float* ddt;           // [B,C] += sum_pos g-dot (acc d) + g u-dot / gain
  // dacc = g d and dacc-dot = g-dot d + g d-dot, as pairs (stride-1 layers) or fp32 (up layers)
  __nv_bfloat16* dacc_hi; __nv_bfloat16* dacc_lo; __nv_bfloat16* dacct_hi; __nv_bfloat16* dacct_lo;
  float* dacc; float* dacct;
  float* g_bias;        // [C] += sum_{b,pos} g-dot, or nullptr
  float* g_noise;       // [B,HW] += sum_c g-dot, or nullptr
};

// act_backward_kernel<true> and its tangent in one pass (lrelu'' = 0): block (chunk, b), 4 channels
// per thread, the seven per-channel sums reduced in shared memory, one atomic per block.
__global__ void __launch_bounds__(256)
act_backward_tangent_kernel(ActBackwardTangent e, int HW, int C, int chunk) {
  __shared__ float4 red[7][256];
  __shared__ float nsum[kActChunk];
  for (int i = threadIdx.x; i < kActChunk; i += 256) nsum[i] = 0.f;
  __syncthreads();
  const int cg = C >> 2, ppar = 256 / cg, tid = threadIdx.x;
  const int p = tid / cg, c4 = tid - p * cg;
  const int b = blockIdx.y;
  const bool active = p < ppar;
  const float inv_gain = 1.f / e.gain;
  float sum[7][4];  // ds_a, ds_b, dd, ds_a-dot, ds_b-dot, dd-dot, bias-dot
#pragma unroll
  for (int q = 0; q < 7; ++q)
#pragma unroll
    for (int k = 0; k < 4; ++k) sum[q][k] = 0.f;
  if (active) {
    auto ld = [](const float* ptr, size_t off, float dflt, float (&o)[4]) {
      if (ptr == nullptr) {
        o[0] = o[1] = o[2] = o[3] = dflt;
        return;
      }
      const float4 t = __ldg(reinterpret_cast<const float4*>(ptr + off));
      o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
    };
    const size_t bc = (size_t)b * C + 4 * c4;
    float d[4], dd[4], bi[4], sa[4], sb[4], ta[4], tb[4];
    ld(e.dcoef, bc, 0.f, d);
    ld(e.ddot, bc, 0.f, dd);
    ld(e.bias, 4 * c4, 0.f, bi);
    ld(e.s_a, bc, 1.f, sa);
    ld(e.s_b, bc, 1.f, sb);
    ld(e.st_a, bc, 0.f, ta);
    ld(e.st_b, bc, 0.f, tb);
    const int end = min(HW, (blockIdx.x + 1) * chunk);
    for (int pos = blockIdx.x * chunk + p; pos < end; pos += ppar) {
      const size_t row = (size_t)b * HW + pos, idx = row * C + 4 * c4;
      float u[4], ud[4], xa[4], xta[4], xb[4], xtb[4];
      ld(e.u, idx, 0.f, u);
      ld(e.u_dot, idx, 0.f, ud);
      ld(e.dx_a, idx, 0.f, xa);
      ld(e.dxt_a, idx, 0.f, xta);
      ld(e.dx_b, idx, 0.f, xb);
      ld(e.dxt_b, idx, 0.f, xtb);
      const float nz = e.noise ? __ldg(e.noise + row) : 0.f;
      float out[4], outt[4], gsum = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float v = lrelu(u[k], kSlope), lg = lrelu_grad(u[k], kSlope), vd = lg * ud[k];
        sum[0][k] = fmaf(xa[k], v, sum[0][k]);
        sum[1][k] = fmaf(xb[k], v, sum[1][k]);
        sum[3][k] += xta[k] * v + xa[k] * vd;
        sum[4][k] += xtb[k] * v + xb[k] * vd;
        const float dv = xa[k] * sa[k] + xb[k] * sb[k];
        const float dvt = (xta[k] * sa[k] + xa[k] * ta[k]) + (xtb[k] * sb[k] + xb[k] * tb[k]);
        const float g = dv * lg * e.gain, gt = dvt * lg * e.gain;
        const float accd = u[k] * inv_gain - nz - bi[k];  // acc d = u/gain - noise - bias
        sum[2][k] = fmaf(g, accd, sum[2][k]);
        sum[5][k] += gt * accd + g * ud[k] * inv_gain;
        sum[6][k] += gt;
        gsum += gt;
        out[k] = g * d[k];
        outt[k] = gt * d[k] + g * dd[k];
      }
      const float4 o4 = make_float4(out[0], out[1], out[2], out[3]);
      const float4 t4 = make_float4(outt[0], outt[1], outt[2], outt[3]);
      const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
      if (e.dacc_hi != nullptr) {
        store_split4(e.dacc_hi, e.dacc_lo, idx, o4, one);
        store_split4(e.dacct_hi, e.dacct_lo, idx, t4, one);
      }
      if (e.dacc != nullptr) {
        *reinterpret_cast<float4*>(e.dacc + idx) = o4;
        *reinterpret_cast<float4*>(e.dacct + idx) = t4;
      }
      if (e.g_noise != nullptr) atomicAdd(&nsum[pos - blockIdx.x * chunk], gsum);
    }
  }
#pragma unroll
  for (int q = 0; q < 7; ++q) red[q][tid] = make_float4(sum[q][0], sum[q][1], sum[q][2], sum[q][3]);
  __syncthreads();
  if (e.g_noise != nullptr) {
    const int p0 = blockIdx.x * chunk, n = min(HW, p0 + chunk) - p0;
    for (int i = tid; i < n; i += 256) e.g_noise[(size_t)b * HW + p0 + i] += nsum[i];
  }
  if (tid < cg) {
    float* dst[7] = {e.ds_a, e.ds_b, e.dd, e.dst_a, e.dst_b, e.ddt, e.g_bias};
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      if (dst[q] == nullptr) continue;
      float4 s = red[q][tid];
      for (int k = 1; k < ppar; ++k) {
        const float4 t = red[q][k * cg + tid];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      float* o = dst[q] + (q == 6 ? 0 : (size_t)b * C) + 4 * tid;
      atomicAdd(o + 0, s.x);
      atomicAdd(o + 1, s.y);
      atomicAdd(o + 2, s.z);
      atomicAdd(o + 3, s.w);
    }
  }
}

// dcoef_backward_kernel and its tangent: with P = sum_o dd d^2 wsq[o,i] and
// Q = sum_o (dd-dot d^2 + 2 dd d d-dot) wsq[o,i]:  ds -= s P,  ds-dot -= s-dot P + s Q
__global__ void dcoef_backward_tangent_kernel(const float* __restrict__ wsq, const float* __restrict__ s,
                                              const float* __restrict__ sdot, const float* __restrict__ dd,
                                              const float* __restrict__ ddt, const float* __restrict__ d,
                                              const float* __restrict__ ddot, int cout, int cin, int B,
                                              float* __restrict__ ds, float* __restrict__ dst) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * cin) return;
  const int b = warp / cin, i = warp % cin;
  float pa = 0.f, qa = 0.f;
  for (int o = lane; o < cout; o += 32) {
    const size_t bo = (size_t)b * cout + o;
    const float dv = d[bo], w = wsq[(size_t)o * cin + i];
    pa = fmaf(dd[bo] * dv * dv, w, pa);
    qa = fmaf(ddt[bo] * dv * dv + 2.f * dd[bo] * dv * ddot[bo], w, qa);
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    pa += __shfl_xor_sync(0xffffffffu, pa, k);
    qa += __shfl_xor_sync(0xffffffffu, qa, k);
  }
  if (lane == 0) {
    ds[warp] -= s[warp] * pa;
    dst[warp] -= sdot[warp] * pa + s[warp] * qa;
  }
}

// wgrad_reduce_kernel with the tangent of the demodulation term: g_w += sum_split part - W sum_b
// [dd-dot d^2 s^2 + 2 dd d d-dot s^2 + 2 dd d^2 s s-dot]; one thread per (co, ci)
__global__ void wgrad_reduce_tangent_kernel(const float* __restrict__ part, int n_split, int taps, int cout,
                                            int cin, const float* __restrict__ w, const float* __restrict__ dd,
                                            const float* __restrict__ ddt, const float* __restrict__ d,
                                            const float* __restrict__ ddot, const float* __restrict__ s,
                                            const float* __restrict__ sdot, int B, float* __restrict__ g_w) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)cout * cin;
  if (i >= n) return;
  const int o = (int)(i / cin), c = (int)(i % cin);
  float dem = 0.f;
  for (int b = 0; b < B; ++b) {
    const size_t bo = (size_t)b * cout + o, bc = (size_t)b * cin + c;
    const float dv = d[bo], sv = s[bc];
    dem += (ddt[bo] * dv * dv + 2.f * dd[bo] * dv * ddot[bo]) * sv * sv + 2.f * dd[bo] * dv * dv * sv * sdot[bc];
  }
  for (int tp = 0; tp < taps; ++tp) {
    float acc = 0.f;
    for (int sp = 0; sp < n_split; ++sp) acc += part[((size_t)sp * taps + tp) * n + i];
    g_w[i * taps + tp] += acc - w[i * taps + tp] * dem;
  }
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

// activation tensor [B,H,W,C] bf16 -> boxes of [1, box_h, 16, 64]
static bool make_act_map(CUtensorMap* tm, const __nv_bfloat16* base, int B, int H, int W, int C,
                         int box_h = kTileH) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {kKBlock, kTileW, (cuuint32_t)box_h, 1};
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

// One convolution launch.  `in` [map_B (default B),H,W,C] pair, weights [taps9][N][C] pair.
static int launch_conv(ConvArgs& a, Pair in, Pair wt, int w_taps, cudaStream_t st, int map_B = 0) {
  if (encode_fn() == nullptr) return fail("cuTensorMapEncodeTiled is not available from this driver");
  a.BN = pick_bn(a.N);
  if (a.BN == 0 || a.C % 8 != 0)  // (TMA: row pitch a multiple of 16 bytes)
    return fail("synthesis conv: unsupported channel counts (Cin %d, Cout %d)", a.C, a.N);
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
      !make_w_map(&tWh, wt.hi, w_taps, a.N, a.C, a.BN) || !make_w_map(&tWl, wt.lo, w_taps, a.N, a.C, a.BN))
    return fail("cuTensorMapEncodeTiled failed (B %d H %d W %d C %d N %d)", a.B, a.H, a.W, a.C, a.N);
  const int smem = kStages * (2 * kATile + 2 * a.BN * 128) + 128 +
                   ((a.mode == kModeRgb && a.skip != nullptr) ? kSkipBytes : 0);
  NFI_CUDA(cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  conv_tc_kernel<<<grid, kConvThreads, smem, st>>>(tAh, tAl, tWh, tWl, a, n_tiles);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// The K split of one weight-gradient GEMM over a DH x DW position domain of B images: fills the
// k-tile counts and split; returns the number of work items.
static int plan_wgrad(WgradArgs& a, int B, int DH, int DW) {
  a.kt_y = (DH + kWgTileH - 1) / kWgTileH;
  a.kt_x = (DW + kWgTileW - 1) / kWgTileW;
  a.kt_img = a.kt_y * a.kt_x;
  a.kt_total = B * a.kt_img;
  a.n_co = (a.cout + 63) / 64;
  a.n_ci = (a.cin + 63) / 64;
  a.chain = kWgChain;
  const int base = a.n_co * a.n_ci * a.taps;
  int n_split = (kWgItems + base - 1) / base;
  const int max_split = (a.kt_total + kWgMinSplit - 1) / kWgMinSplit;
  if (n_split > max_split) n_split = max_split;
  if (n_split < 1) n_split = 1;
  a.split_len = (a.kt_total + n_split - 1) / n_split;
  a.n_split = (a.kt_total + a.split_len - 1) / a.split_len;
  return base * a.n_split;
}

// One weight-gradient GEMM (plan_wgrad'ed `a`): G [gB,gH,gW,g_channels (default cout)] and
// X [B,xH,xW,cin] pairs.
static int launch_wgrad(WgradArgs& a, Pair g, int gB, int gH, int gW, Pair x, int B, int xH, int xW,
                        cudaStream_t st, int g_channels = 0) {
  if (encode_fn() == nullptr) return fail("cuTensorMapEncodeTiled is not available from this driver");
  const int n_items = a.n_co * a.n_ci * a.taps * a.n_split;
  if (g_channels == 0) g_channels = a.cout;
  CUtensorMap tGh, tGl, tXh, tXl;
  if (!make_act_map(&tGh, g.hi, gB, gH, gW, g_channels, kWgTileH) ||
      !make_act_map(&tGl, g.lo, gB, gH, gW, g_channels, kWgTileH) ||
      !make_act_map(&tXh, x.hi, B, xH, xW, a.cin, kWgTileH) ||
      !make_act_map(&tXl, x.lo, B, xH, xW, a.cin, kWgTileH))
    return fail("cuTensorMapEncodeTiled failed (weight gradient, Cout %d Cin %d)", a.cout, a.cin);
  const int smem = kWgStages * kWgStage + 128;
  NFI_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = n_items < 2 * sm_count() ? n_items : 2 * sm_count();
  wgrad_tc_kernel<<<grid, kWgThreads, smem, st>>>(tGh, tGl, tXh, tXl, a, n_items);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// ---- conv descriptors: one per GEMM shape the network runs on conv_tc_kernel, with its phases,
// taps, mode and output extents; the caller sets the epilogue's pointers ----
static ConvArgs conv_args(int B, int C, int N, int H, int W, int mode) {
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.B = B; a.C = C; a.N = N; a.H = H; a.W = W;
  a.mode = mode;
  return a;
}
// The stride-1 3x3 conv (pad 1, cross-correlation) of [B,H,W,C] into N channels; RAW writes
// [B,H,W,N].  `adjoint` flips the taps: conv^T, the data gradient against prep_weights_t_kernel's W.
static ConvArgs conv3x3_args(int B, int C, int N, int H, int W, int mode, bool adjoint = false) {
  ConvArgs a = conv_args(B, C, N, H, W, mode);
  a.n_phases = 1;
  a.ph_taps[0] = 9;
  a.ph_DH[0] = H;
  a.ph_DW[0] = W;
  const int sign = adjoint ? -1 : 1;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      a.tap_dy[t] = sign * (ky - 1);
      a.tap_dx[t] = sign * (kx - 1);
      a.tap_w[t] = t;
    }
  if (mode == kModeRaw) { a.out_H = H; a.out_W = W; a.out_stride = 1; }
  return a;
}
// conv_transpose2d(stride 2) of [B,h,h,C] into the (2h+1)^2 raw result (RAW; fir_act_kernel filters
// it): out[2i+ky, 2j+kx] += x[i,j] W[ky,kx].  Output parity (py,px) takes the taps with
// ky = py (mod 2), kx = px (mod 2); position (a,b) of the phase reads x[a - ky/2, b - kx/2].
static ConvArgs conv_up_args(int B, int C, int N, int h) {
  ConvArgs a = conv_args(B, C, N, h, h, kModeRaw);
  a.n_phases = 4;
  int t = 0;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      const int p = py * 2 + px;
      a.ph_tap0[p] = t;
      a.ph_DH[p] = py ? h : h + 1;
      a.ph_DW[p] = px ? h : h + 1;
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
  a.out_H = a.out_W = 2 * h + 1;
  a.out_stride = 2;
  return a;
}
// The adjoint of conv_up_args: the stride-2 correlation with W0 as 9 stride-1 taps over the four
// parity phases of the raw gradient, phase (py,px) at image offset (2py+px) nimg of a
// [4 nimg, h+1, h+1, C] pair (fir_adjoint_kernel; nimg = B, or 2B with the tangent stacked): tap
// (ky,kx) reads phase (ky%2, kx%2) at offset (ky/2, kx/2).  RAW into [nimg,h,h,N]; the caller's
// activation map spans all 4 nimg images.
static ConvArgs conv_up_adjoint_args(int nimg, int C, int N, int h) {
  ConvArgs a = conv_args(nimg, C, N, h + 1, h + 1, kModeRaw);
  a.n_phases = 1;
  a.ph_taps[0] = 9;
  a.ph_DH[0] = h;
  a.ph_DW[0] = h;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      a.tap_dy[t] = ky / 2;
      a.tap_dx[t] = kx / 2;
      a.tap_w[t] = t;
      a.tap_img[t] = ((ky & 1) * 2 + (kx & 1)) * nimg;
    }
  a.out_H = h; a.out_W = h; a.out_stride = 1;
  return a;
}
// ToRGB, the 1x1 conv at resolution res: forward (kModeRgb) from the layer's [B,res,res,C] input
// into the N = 96 image channels, or its adjoint (kModeRaw) from the image gradient into
// [B,res,res,N]
static ConvArgs torgb_args(int B, int C, int N, int res, int mode) {
  ConvArgs a = conv_args(B, C, N, res, res, mode);
  a.n_phases = 1;
  a.ph_taps[0] = 1;
  a.ph_DH[0] = res;
  a.ph_DW[0] = res;
  if (mode == kModeRaw) { a.out_H = res; a.out_W = res; a.out_stride = 1; }
  return a;
}

// ---- tap tables of the weight GEMMs (plan_wgrad fills the rest) ----
static WgradArgs wgrad_args(int cout, int cin, int taps) {
  WgradArgs a;
  memset(&a, 0, sizeof(a));
  a.cout = cout; a.cin = cin; a.taps = taps;
  return a;
}
// ToRGB: dimg against the layer's input at the same position
static WgradArgs torgb_wgrad(int cout, int cin) { return wgrad_args(cout, cin, 1); }
// A stride-1 3x3 conv: the output gradient at p against the input at p + (ky - 1, kx - 1)
static WgradArgs conv3x3_wgrad(int cout, int cin) {
  WgradArgs a = wgrad_args(cout, cin, 9);
  for (int t = 0; t < 9; ++t) {
    a.x_dy[t] = t / 3 - 1;
    a.x_dx[t] = t % 3 - 1;
  }
  return a;
}
// conv1 (stride 1): dacc against x~
static WgradArgs conv1_wgrad(int c) { return conv3x3_wgrad(c, c); }
// conv0 (up): the raw gradient at (2i+ky, 2j+kx) is phase (ky%2, kx%2) at (i + ky/2, j + kx/2), the
// phases stacked as in conv_up_adjoint_args over nimg images each, against x~ at (i, j)
static WgradArgs conv0_wgrad(int cout, int cin, int nimg) {
  WgradArgs a = wgrad_args(cout, cin, 9);
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      a.a_dy[t] = ky / 2;
      a.a_dx[t] = kx / 2;
      a.a_img[t] = ((ky & 1) * 2 + (kx & 1)) * nimg;
    }
  return a;
}

static int check_params(const nfi_synth_params& P) {
  const int R = P.img_resolution;
  int nb = 0;
  for (int r = 4; r <= R; r <<= 1) ++nb;
  if (R < 8 || (R & (R - 1)) || nb != P.num_blocks || nb > NFI_SYNTH_MAX_BLOCKS)
    return fail("synthesis: img_resolution %d / num_blocks %d inconsistent", R, P.num_blocks);
  if (P.img_channels != 96) return fail("synthesis: img_channels must be 96 (3 planes x 32), got %d", P.img_channels);
  if (P.num_ws < 2 * nb) return fail("synthesis: ws has %d rows, need %d", P.num_ws, 2 * nb);
  for (int i = 0; i < nb; ++i)
    if (P.channels[i] % 32 != 0 || pick_bn(P.channels[i]) == 0)
      return fail("synthesis: block %d has %d channels (need a multiple of 32 that tiles)", i, P.channels[i]);
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
  Pair w0[NFI_SYNTH_MAX_BLOCKS], w1[NFI_SYNTH_MAX_BLOCKS];  // [tap][Cout][Cin] pairs of the forward
  int row0[NFI_SYNTH_MAX_BLOCKS], row1[NFI_SYNTH_MAX_BLOCKS], row_rgb[NFI_SYNTH_MAX_BLOCKS];
};

// Runs (or, with dry, only lays out) the whole network.  With `sv`, the forward also stores every
// layer's pre-activation u (the save mode) and `sv` receives the pointers the backward reads.
static int run(const nfi_synth_params& P, Bump& ws, cudaStream_t st, bool dry, Saved* sv = nullptr) {
  const int B = P.batch, nb = P.num_blocks, D = P.w_dim;
  const float sqrt2 = 1.4142135623730951f;

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
      if (i) sv->w0[i] = w0[i];
      sv->w1[i] = w1[i];
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
        ConvArgs a = conv_up_args(B, cin, cout, hin);
        a.out_raw = raw;
        const int rc = launch_conv(a, x, w0[i], 9, st);
        if (rc) return rc;
        ActEpilogue e;
        memset(&e, 0, sizeof(e));
        e.dcoef = dco0[i]; e.noise = P.conv0[i].noise; e.bias = P.conv0[i].bias; e.gain = sqrt2;
        e.slope = 0.2f;
        e.style_a = style1[i]; e.a_hi = y.hi; e.a_lo = y.lo;
        e.u_out = sv ? sv->u0[i] : nullptr;
        const size_t total = (size_t)B * (res / 2) * (res / 2) * (cout / 4);
        fir_act_kernel<<<flat_grid(total), 256, 0, st>>>(raw, B, res, res, cout, e);
        NFI_CUDA(cudaGetLastError());
      }
      x = y;
    }
    // conv1 (stride 1) with the fused ACT epilogue; consumers: next block's conv0 and this ToRGB
    Pair xn = {nullptr, nullptr};
    if (!last) xn = ws.pair((size_t)B * res * res * cout);
    Pair xr = ws.pair((size_t)B * res * res * cout);
    if (!dry) {
      ConvArgs a = conv3x3_args(B, cout, cout, res, res, kModeAct);
      a.act.dcoef = dco1[i]; a.act.noise = P.conv1[i].noise; a.act.bias = P.conv1[i].bias;
      a.act.gain = sqrt2;
      a.act.slope = 0.2f;
      a.act.style_a = style_rgb[i]; a.act.a_hi = xr.hi; a.act.a_lo = xr.lo;
      if (!last) { a.act.style_b = style0[i + 1]; a.act.b_hi = xn.hi; a.act.b_lo = xn.lo; }
      a.act.u_out = sv ? sv->u1[i] : nullptr;
      const int rc = launch_conv(a, x, w1[i], 9, st);
      if (rc) return rc;
    }
    // ToRGB (1x1, K = cout) + bias + upsampled running image
    float* img = last ? nullptr : ws.take((size_t)B * res * res * P.img_channels);
    if (!dry) {
      ConvArgs a = torgb_args(B, cout, P.img_channels, res, kModeRgb);
      a.act.bias = P.torgb[i].bias;
      a.skip = img_prev; a.img = img; a.planes = last ? P.planes : nullptr;
      const int rc = launch_conv(a, xr, wrgb[i], 1, st);
      if (rc) return rc;
    }
    img_prev = img;
    x = xn;
  }
  return 0;
}

// A sizer: 0 for params check_params refuses, else what `layout` takes from a dry Bump plus the
// 1024 bytes an entry may lose aligning the caller's pointer
template <class Layout>
static size_t sized(const nfi_synth_params& P, Layout layout) {
  if (check_params(P)) return 0;
  Bump b{nullptr, 0, 0};
  layout(b);
  return b.off + 1024;
}

size_t workspace_bytes(const nfi_synth_params& P) {
  return sized(P, [&](Bump& b) { run(P, b, nullptr, true); });
}

int forward(const nfi_synth_params& P, cudaStream_t st) {
  const int rc = check_params(P);
  if (rc) return rc;
  if (P.ws == nullptr || P.const_input == nullptr || P.planes == nullptr || P.workspace == nullptr)
    return fail("synthesis: ws, const_input, planes and workspace must be set");
  const size_t need = workspace_bytes(P);
  if (P.workspace_bytes < need)
    return fail("synthesis: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  Bump b = aligned_bump(P.workspace, P.workspace_bytes);
  return run(P, b, st, false);
}

// ---- backward ----
// The scratch of the backward walk (run_backward) and of its tangent (run_hvp), for `copies` stacked
// copies of every quantity the walk derives from ws: 1, or 2 for [q; q-dot] on 2B images.  Reused
// across blocks (stream order keeps the reuse safe): bufA holds g_rgb, then dx~ of conv1, then the
// raw-gradient phases of conv0; bufB the dacc of conv1 (pair), then of conv0 (fp32); bufC dx~ of
// conv0 until the previous block's conv1 has consumed it.
struct BackwardScratch {
  float *bufA, *bufB, *bufC;
  float* dimg[2];  // the running image's gradient, alternately per block (one copy: not from ws)
  Pair dimg_p;
  float* sums;     // the per-(b, channel) sums of every copy, zeroed once
  size_t n_sums;
  float *ds0[2][NFI_SYNTH_MAX_BLOCKS], *ds1[2][NFI_SYNTH_MAX_BLOCKS], *dsr[2][NFI_SYNTH_MAX_BLOCKS];
  float *dd0[2][NFI_SYNTH_MAX_BLOCKS], *dd1[2][NFI_SYNTH_MAX_BLOCKS];  // [copy][block]
  Pair wt0[NFI_SYNTH_MAX_BLOCKS], wt1[NFI_SYNTH_MAX_BLOCKS], wtr[NFI_SYNTH_MAX_BLOCKS];  // W^T pairs
  Pair xt;         // the layer input x~ of the current weight GEMM, `copies` deep (or none)
  float* part;     // the weight GEMMs' partials (or none)
};

// Takes the scratch from `ws`; x~ with `take_xt`, the partials with `plan_parts`.  The optional
// buffers come last, so the ones every walk uses keep their places.
static BackwardScratch backward_scratch(const nfi_synth_params& P, Bump& ws, int copies, bool take_xt,
                                        bool plan_parts) {
  const int B = P.batch, nb = P.num_blocks, R = P.img_resolution, NI = P.img_channels;
  BackwardScratch s;
  memset(&s, 0, sizeof(s));
  int cmax = 0;
  for (int i = 0; i < nb; ++i) cmax = P.channels[i] > cmax ? P.channels[i] : cmax;
  const size_t full = (size_t)copies * B * R * R * cmax;
  const size_t phases = (size_t)4 * copies * B * (R / 2 + 1) * (R / 2 + 1) * cmax;
  s.bufA = ws.take(full > phases ? full : phases);  // (the HVP: also the tangent conv's raw output)
  s.bufB = ws.take(full);
  s.bufC = ws.take((size_t)copies * B * (R / 2) * (R / 2) * cmax);
  s.dimg[0] = ws.take((size_t)B * R * R * NI);
  s.dimg[1] = ws.take((size_t)B * R * R * NI);
  s.dimg_p = ws.pair((size_t)B * R * R * NI);
  size_t small = 0;
  for (int i = 0; i < nb; ++i) small += (size_t)B * (4 * P.channels[i] + (i ? P.channels[i - 1] : 0));
  s.n_sums = copies * small;
  s.sums = ws.take(s.n_sums);
  float* q = s.sums;
  for (int k = 0; k < copies; ++k)
    for (int i = 0; i < nb; ++i) {
      const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
      s.ds0[k][i] = q; q += (size_t)B * ci;
      s.ds1[k][i] = q; q += (size_t)B * c;
      s.dsr[k][i] = q; q += (size_t)B * c;
      s.dd0[k][i] = q; q += (size_t)B * c;
      s.dd1[k][i] = q; q += (size_t)B * c;
    }
  for (int i = 0; i < nb; ++i) {
    const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
    if (i) s.wt0[i] = ws.pair((size_t)9 * c * ci);
    s.wt1[i] = ws.pair((size_t)9 * c * c);
    s.wtr[i] = ws.pair((size_t)NI * c);
  }
  if (take_xt) s.xt = ws.pair(full);
  if (plan_parts) {  // the largest GEMM's; ToRGB's runs on one copy (dimg does not depend on ws)
    size_t pmax = 0;
    auto need = [&](WgradArgs a, int nimg, int D_) {
      plan_wgrad(a, nimg, D_, D_);
      const size_t n = (size_t)a.n_split * a.taps * a.cout * a.cin;
      pmax = n > pmax ? n : pmax;
    };
    for (int i = 0; i < nb; ++i) {
      const int res = 4 << i, c = P.channels[i];
      need(torgb_wgrad(NI, c), B, res);
      need(conv1_wgrad(c), copies * B, res);
      if (i) need(conv0_wgrad(c, P.channels[i - 1], copies * B), copies * B, res / 2);
    }
    s.part = ws.take(pmax);
  }
  return s;
}

// The walk's operands that do not depend on it: every layer's W^T pair, and the planes' gradient
// as the last block's image gradient dimg[0] (fp32 and pair)
static int prep_backward(const nfi_synth_params& P, const float* g_planes, const BackwardScratch& s, cudaStream_t st) {
  const int B = P.batch, R = P.img_resolution, NI = P.img_channels;
  auto prep_t = [&](const float* w, int cout, int cin, int taps, Pair out) {
    return prep_weights(w, cout, cin, taps, cin * taps, 1.f, kTapCiCo, out, st);
  };
  for (int i = 0; i < P.num_blocks; ++i) {
    const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
    if (i > 0)
      if (const int rc = prep_t(P.conv0[i].weight, c, ci, 9, s.wt0[i])) return rc;
    if (const int rc = prep_t(P.conv1[i].weight, c, c, 9, s.wt1[i])) return rc;
    if (const int rc = prep_t(P.torgb[i].weight, NI, c, 1, s.wtr[i])) return rc;
  }
  planes_grad_kernel<<<flat_grid((size_t)B * R * R * NI), 256, 0, st>>>(g_planes, B, R, s.dimg[0],
                                                                        s.dimg_p.hi, s.dimg_p.lo);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// Walks the blocks from the last to the first.
// With `PG` (the parameter backward) the same launches run, act_backward_kernel<true> in place of
// <false>, and each layer's weight GEMM runs while its gradient operand is still in scratch: ToRGB
// on dimg before the running image's adjoint overwrites it, conv1 on its dacc pair, conv0 on the
// raw-gradient phases.  It also takes the rebuilt layer input x~ and the GEMM partials.
static int run_backward(const nfi_synth_params& P, const nfi_synth_grads& G, const Saved& sv, Bump& ws,
                        cudaStream_t st, bool dry, const nfi_synth_param_grads* PG = nullptr) {
  const int B = P.batch, nb = P.num_blocks, D = P.w_dim, NI = P.img_channels;
  const float sqrt2 = 1.4142135623730951f;
  const BackwardScratch s = backward_scratch(P, ws, 1, PG != nullptr, PG != nullptr);
  if (dry) return 0;
  float *const bufA = s.bufA, *const bufB = s.bufB, *const bufC = s.bufC, *const part = s.part;
  const auto& dimg = s.dimg;
  const auto &wt0 = s.wt0, &wt1 = s.wt1, &wtr = s.wtr;
  const auto &ds0 = s.ds0[0], &ds1 = s.ds1[0], &dsr = s.dsr[0], &dd0 = s.dd0[0], &dd1 = s.dd1[0];
  const Pair dimg_p = s.dimg_p, xt = s.xt;

  NFI_CUDA(cudaMemsetAsync(s.sums, 0, s.n_sums * sizeof(float), st));
  if (const int rc = prep_backward(P, G.g_planes, s, st)) return rc;

  auto act_backward = [&](ActBackward& e, int HW, int C) -> int {
    if (C % 4 != 0 || C / 4 > 256) return fail("synthesis backward: %d channels unsupported", C);
    const int chunk = kActChunk;
    dim3 grid((unsigned)((HW + chunk - 1) / chunk), (unsigned)B);
    if (PG)
      act_backward_kernel<true><<<grid, 256, 0, st>>>(e, HW, C, chunk);
    else
      act_backward_kernel<false><<<grid, 256, 0, st>>>(e, HW, C, chunk);
    NFI_CUDA(cudaGetLastError());
    return 0;
  };
  auto to_ws = [&](const float* ds, const nfi_synth_layer& L, int cin, int row, float gain) {
    styles_backward_kernel<<<blocks((size_t)B * D, 256), 256, 0, st>>>(
        ds, L.affine_w, cin, D, B, gain / sqrtf((float)D), G.g_ws + (size_t)row * D, P.num_ws * D);
  };
  // ---- parameter backward (PG only) ----
  auto affine = [&](const float* ds, const nfi_synth_layer_grads& L, int cin, int row, float gain) {
    if (L.g_affine_w == nullptr && L.g_affine_b == nullptr) return;
    affine_backward_kernel<<<blocks((size_t)cin * D, 256), 256, 0, st>>>(
        ds, P.ws + (size_t)row * D, P.num_ws * D, B, cin, D, gain / sqrtf((float)D), gain, L.g_affine_w,
        L.g_affine_b);
  };
  auto restyle = [&](const float* u, const float* s, int HW, int C) {
    restyle_kernel<<<flat_grid((size_t)B * HW * C / 4), 256, 0, st>>>(u, s, B, HW, C, xt.hi, xt.lo);
  };
  // plan, GEMM into the partials, then the fixed-order sum (+ demodulation term where dd is set)
  auto wgrad = [&](WgradArgs& a, Pair g, int gB, int gH, int D_, const float* w, const float* dd,
                   const float* d, const float* s, float* g_w) -> int {
    plan_wgrad(a, B, D_, D_);
    a.part = part;
    if (const int rc = launch_wgrad(a, g, gB, gH, gH, xt, B, D_, D_, st)) return rc;
    wgrad_reduce_kernel<<<blocks((size_t)a.cout * a.cin, 256), 256, 0, st>>>(
        part, a.n_split, a.taps, a.cout, a.cin, w, dd, d, s, B, g_w);
    NFI_CUDA(cudaGetLastError());
    return 0;
  };

  int cur = 0;  // dimg[cur] is the gradient of block i's running image
  for (int i = nb - 1; i >= 0; --i) {
    const int res = 4 << i, c = P.channels[i], ci = i ? P.channels[i - 1] : 0, HW = res * res;
    const bool last = (i == nb - 1);
    // ToRGB: g = dimg Wrgb^T  [B,res,res,c] -> bufA
    {
      ConvArgs a = torgb_args(B, NI, c, res, kModeRaw);
      a.out_raw = bufA;
      const int rc = launch_conv(a, dimg_p, wtr[i], 1, st);
      if (rc) return rc;
    }
    if (PG) {  // ToRGB bias and weight: sum dimg, and dimg against x~ = lrelu(u1) s_rgb
      const nfi_synth_layer_grads& L = PG->torgb[i];
      if (L.g_bias != nullptr) {
        const size_t rows = (size_t)B * HW;
        colsum_kernel<<<blocks(rows, kActChunk), 256, 0, st>>>(dimg[cur], rows, NI, kActChunk, L.g_bias);
      }
      if (L.g_weight != nullptr) {
        restyle(sv.u1[i], sv.style_rgb[i], HW, c);
        WgradArgs a = torgb_wgrad(NI, c);
        if (int rc = wgrad(a, dimg_p, B, res, res, P.torgb[i].weight, nullptr, nullptr, nullptr, L.g_weight))
          return rc;
      }
    }
    if (i) {  // the running image's gradient one block down (the GEMM above has read dimg_p)
      const int h = res / 2;
      upsample_adjoint_kernel<<<flat_grid((size_t)B * h * h * NI), 256, 0, st>>>(
          dimg[cur], B, h, h, NI, dimg[cur ^ 1], dimg_p.hi, dimg_p.lo);
      NFI_CUDA(cudaGetLastError());
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
      if (PG) {
        e.g_bias = PG->conv1[i].g_bias;
        e.g_noise = P.conv1[i].noise ? PG->conv1[i].g_noise : nullptr;
      }
      if (int rc = act_backward(e, HW, c)) return rc;
      to_ws(dsr[i], P.torgb[i], c, sv.row_rgb[i], 1.f / sqrtf((float)c));
      if (PG) affine(dsr[i], PG->torgb[i], c, sv.row_rgb[i], 1.f / sqrtf((float)c));
      if (!last) {
        const int cn = P.channels[i + 1];
        dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
            sv.wsq0[i + 1], sv.style0[i + 1], dd0[i + 1], sv.dco0[i + 1], cn, c, B, ds0[i + 1]);
        to_ws(ds0[i + 1], P.conv0[i + 1], c, sv.row0[i + 1], 1.f);
        if (PG) affine(ds0[i + 1], PG->conv0[i + 1], c, sv.row0[i + 1], 1.f);
      }
      // dx~ of conv1 = conv^T(dacc, W1) -> bufA
      ConvArgs a = conv3x3_args(B, c, c, res, res, kModeRaw, true);
      a.out_raw = bufA;
      const int rc = launch_conv(a, pb, wt1[i], 9, st);
      if (rc) return rc;
      if (PG && PG->conv1[i].g_weight != nullptr) {  // dacc against x~ = lrelu(u0) s1 (const s1)
        if (i)
          restyle(sv.u0[i], sv.style1[i], HW, c);
        else
          const_input_kernel<<<blocks((size_t)B * 16 * c, 256), 256, 0, st>>>(P.const_input, sv.style1[0],
                                                                             B, c, xt.hi, xt.lo);
        WgradArgs w = conv1_wgrad(c);
        if (int rc2 = wgrad(w, pb, B, res, res, P.conv1[i].weight, dd1[i], sv.dco1[i], sv.style1[i],
                            PG->conv1[i].g_weight))
          return rc2;
      }
    }
    if (i == 0) {
      const_ds_kernel<<<blocks((size_t)B * c, 256), 256, 0, st>>>(bufA, P.const_input, B, c, ds1[0]);
      if (PG && PG->g_const != nullptr)
        const_grad_kernel<<<blocks((size_t)c * 16, 256), 256, 0, st>>>(bufA, sv.style1[0], B, c, PG->g_const);
      dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
          sv.wsq1[0], sv.style1[0], dd1[0], sv.dco1[0], c, c, B, ds1[0]);
      to_ws(ds1[0], P.conv1[0], c, sv.row1[0], 1.f);
      if (PG) affine(ds1[0], PG->conv1[0], c, sv.row1[0], 1.f);
      NFI_CUDA(cudaGetLastError());
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
      if (PG) {
        e.g_bias = PG->conv0[i].g_bias;
        e.g_noise = P.conv0[i].noise ? PG->conv0[i].g_noise : nullptr;
      }
      if (int rc = act_backward(e, HW, c)) return rc;
      dcoef_backward_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(
          sv.wsq1[i], sv.style1[i], dd1[i], sv.dco1[i], c, c, B, ds1[i]);
      to_ws(ds1[i], P.conv1[i], c, sv.row1[i], 1.f);
      if (PG) affine(ds1[i], PG->conv1[i], c, sv.row1[i], 1.f);
    }
    // FIR adjoint -> the four parity phases of the raw gradient (pair in bufA), then the
    // stride-2 correlation with W0 as 9 stride-1 taps over them -> dx~ of conv0 in bufC
    {
      const int h = res / 2;
      Pair ph = {reinterpret_cast<__nv_bfloat16*>(bufA),
                 reinterpret_cast<__nv_bfloat16*>(bufA) + (size_t)4 * B * (h + 1) * (h + 1) * c};
      fir_adjoint_kernel<<<flat_grid((size_t)4 * B * (h + 1) * (h + 1) * (c / 4)), 256, 0, st>>>(
          bufB, B, res, res, c, ph.hi, ph.lo);
      NFI_CUDA(cudaGetLastError());
      if (PG && PG->conv0[i].g_weight != nullptr) {
        // raw gradient at (2i+ky, 2j+kx) = phase (ky%2, kx%2) at (i + ky/2, j + kx/2), against
        // x~ = lrelu(u1 of block i-1) s0 on the low-resolution grid
        restyle(sv.u1[i - 1], sv.style0[i], h * h, ci);
        WgradArgs w = conv0_wgrad(c, ci, B);
        if (int rc = wgrad(w, ph, 4 * B, h + 1, h, P.conv0[i].weight, dd0[i], sv.dco0[i], sv.style0[i],
                           PG->conv0[i].g_weight))
          return rc;
      }
      ConvArgs a = conv_up_adjoint_args(B, c, ci, h);
      a.out_raw = bufC;
      const int rc = launch_conv(a, ph, wt0[i], 9, st, 4 * B);
      if (rc) return rc;
    }
  }
  NFI_CUDA(cudaGetLastError());
  return 0;
}

static int saved_layout(const nfi_synth_params& P, Bump& b, Saved& sv) {
  return run(P, b, nullptr, true, &sv);
}

// The saved forward and, after it, the backward's scratch (with PG, the parameter backward's)
static size_t backward_bytes(const nfi_synth_params& P, const nfi_synth_param_grads* PG) {
  return sized(P, [&](Bump& b) {
    Saved sv{};
    saved_layout(P, b, sv);
    run_backward(P, nfi_synth_grads{}, sv, b, nullptr, true, PG);
  });
}

size_t saved_workspace_bytes(const nfi_synth_params& P) { return backward_bytes(P, nullptr); }

size_t param_workspace_bytes(const nfi_synth_params& P) {
  const nfi_synth_param_grads pg{};
  return backward_bytes(P, &pg);
}

static int check_saved(const nfi_synth_params& P) {
  const int rc = check_params(P);
  if (rc) return rc;
  if (P.ws == nullptr || P.const_input == nullptr || P.planes == nullptr || P.workspace == nullptr)
    return fail("synthesis: ws, const_input, planes and workspace must be set");
  const size_t need = saved_workspace_bytes(P);
  if (P.workspace_bytes < need)
    return fail("synthesis: saved workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  return 0;
}

// The prologue of every entry that uses the saved workspace: the checks (the params and the saved
// workspace's size; g_planes and g_ws where G is given; the parameter backward's larger workspace
// with `param_ws`), then the Bump over the aligned workspace and, where `sv` is given, the saved
// forward's pointers, which leave the Bump past the saved forward.
static int open_saved(const nfi_synth_params& P, const nfi_synth_grads* G, bool param_ws, Bump& b, Saved* sv) {
  if (const int rc = check_saved(P)) return rc;
  if (G != nullptr && (G->g_planes == nullptr || G->g_ws == nullptr))
    return fail("synthesis backward: g_planes and g_ws must be set");
  if (param_ws) {
    const size_t need = param_workspace_bytes(P);
    if (P.workspace_bytes < need)
      return fail("synthesis parameter backward: workspace too small (%zu < %zu bytes)", P.workspace_bytes, need);
  }
  b = aligned_bump(P.workspace, P.workspace_bytes);
  if (sv == nullptr) return 0;
  *sv = Saved{};
  return saved_layout(P, b, *sv);
}

int forward_saved(const nfi_synth_params& P, cudaStream_t st) {
  Bump b;
  if (const int rc = open_saved(P, nullptr, false, b, nullptr)) return rc;
  Saved sv{};
  return run(P, b, st, false, &sv);
}

int backward(const nfi_synth_params& P, const nfi_synth_grads& G, cudaStream_t st) {
  Bump b;
  Saved sv;
  if (const int rc = open_saved(P, &G, false, b, &sv)) return rc;
  return run_backward(P, G, sv, b, st, false);
}

int saved_preactivation(const nfi_synth_params& P, int block, int which, float* out, cudaStream_t st) {
  Bump b;
  Saved sv;
  if (const int rc = open_saved(P, nullptr, false, b, &sv)) return rc;
  if (block < 0 || block >= P.num_blocks || (which != 0 && which != 1) || (which == 0 && block == 0))
    return fail("synthesis pre-activation: no layer (block %d, which %d)", block, which);
  if (out == nullptr) return fail("synthesis pre-activation: out must be set");
  const int res = 4 << block;
  const size_t n = (size_t)P.batch * res * res * P.channels[block];
  NFI_CUDA(cudaMemcpyAsync(out, which ? sv.u1[block] : sv.u0[block], n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int backward_params(const nfi_synth_params& P, const nfi_synth_grads& G, const nfi_synth_param_grads& PG,
                    cudaStream_t st) {
  Bump b;
  Saved sv;
  if (const int rc = open_saved(P, &G, true, b, &sv)) return rc;
  return run_backward(P, G, sv, b, st, false, &PG);
}


// ---- path-length HVP (nfi_synthesis_backward_hvp) ----
// Scratch of its own (the saved workspace is only read).  The tangent forward keeps s-dot, d-dot
// and u-dot of every layer; the walk then runs run_backward's launches on 2B stacked images where
// a quantity and its tangent meet the same operand: the data-gradient GEMMs on [dacc; dacc-dot]
// against W^T, the weight GEMMs on [dacc; dacc-dot] against [x~-dot; x~] (one sum over 2B images
// is the product rule's two terms).  Buffers as in run_backward, with room for 2B images.
static int run_hvp(const nfi_synth_params& P, const nfi_synth_hvp& H, const Saved& sv, Bump& ws,
                   cudaStream_t st, bool dry, const nfi_synth_param_grads* PG) {
  const int B = P.batch, B2 = 2 * B, nb = P.num_blocks, D = P.w_dim, NI = P.img_channels;
  const float sqrt2 = 1.4142135623730951f;
  // xt is [x~-dot; x~]: the tangent conv's input, the weight GEMMs' X
  const BackwardScratch s = backward_scratch(P, ws, 2, true, PG != nullptr);
  // u-dot of every layer, and the style and dcoef tangents
  float *ud0[NFI_SYNTH_MAX_BLOCKS] = {nullptr}, *ud1[NFI_SYNTH_MAX_BLOCKS];
  for (int i = 0; i < nb; ++i) {
    const size_t n = (size_t)B * (4 << i) * (4 << i) * P.channels[i];
    if (i) ud0[i] = ws.take(n);
    ud1[i] = ws.take(n);
  }
  float *sd0[NFI_SYNTH_MAX_BLOCKS], *sd1[NFI_SYNTH_MAX_BLOCKS], *sdr[NFI_SYNTH_MAX_BLOCKS];
  float *ddot0[NFI_SYNTH_MAX_BLOCKS], *ddot1[NFI_SYNTH_MAX_BLOCKS];
  for (int i = 0; i < nb; ++i) {
    const int c = P.channels[i], ci = i ? P.channels[i - 1] : 0;
    sd0[i] = i ? ws.take((size_t)B * ci) : nullptr;
    ddot0[i] = i ? ws.take((size_t)B * c) : nullptr;
    sd1[i] = ws.take((size_t)B * c);
    ddot1[i] = ws.take((size_t)B * c);
    sdr[i] = ws.take((size_t)B * c);
  }
  if (dry) return 0;
  float *const bufA = s.bufA, *const bufB = s.bufB, *const bufC = s.bufC, *const part = s.part;
  const auto& dimg = s.dimg;
  const auto &wt0 = s.wt0, &wt1 = s.wt1, &wtr = s.wtr;
  const auto &ds0 = s.ds0, &ds1 = s.ds1, &dsr = s.dsr, &dd0 = s.dd0, &dd1 = s.dd1;  // [0]: q, [1]: q-dot
  const Pair dimg_p = s.dimg_p, xt = s.xt;

  NFI_CUDA(cudaMemsetAsync(s.sums, 0, s.n_sums * sizeof(float), st));
  // ---- tangent forward ----
  auto style_dot = [&](const nfi_synth_layer& L, int c, int row, float gain, float* out) {
    styles_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(H.t_ws + (size_t)row * D, P.num_ws * D, D,
                                                                   L.affine_w, nullptr, c, B, gain, out);
  };
  auto restyle_dot = [&](const float* u, const float* ud, const float* s, const float* sdot, int HW, int C,
                         Pair dst) {
    restyle_tangent_kernel<<<flat_grid((size_t)B * HW * C / 4), 256, 0, st>>>(u, ud, s, sdot, B, HW, C, dst.hi,
                                                                             dst.lo);
  };
  auto tangent_epi = [&](const nfi_synth_layer& L, const float* d, const float* ddot, const float* u,
                         float* udot) {
    TangentEpilogue e;
    e.dcoef = d; e.ddot = ddot; e.noise = L.noise; e.bias = L.bias; e.u = u; e.gain = sqrt2; e.u_dot = udot;
    return e;
  };
  for (int i = 0; i < nb; ++i) {
    const int res = 4 << i, c = P.channels[i], ci = i ? P.channels[i - 1] : 0, HW = res * res;
    if (i) {
      style_dot(P.conv0[i], ci, sv.row0[i], 1.f, sd0[i]);
      dcoef_tangent_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(sv.wsq0[i], sv.style0[i], sd0[i],
                                                                           sv.dco0[i], c, ci, B, ddot0[i]);
    }
    style_dot(P.conv1[i], c, sv.row1[i], 1.f, sd1[i]);
    dcoef_tangent_kernel<<<blocks((size_t)B * c * 32, 256), 256, 0, st>>>(sv.wsq1[i], sv.style1[i], sd1[i],
                                                                         sv.dco1[i], c, c, B, ddot1[i]);
    style_dot(P.torgb[i], c, sv.row_rgb[i], 1.f / sqrtf((float)c), sdr[i]);
    if (i) {  // conv0: x~-dot on the low-resolution grid, the four phase GEMMs, FIR + tangent epilogue
      const int h = res / 2;
      restyle_dot(sv.u1[i - 1], ud1[i - 1], sv.style0[i], sd0[i], h * h, ci, xt);
      ConvArgs a = conv_up_args(B, ci, c, h);
      a.out_raw = bufA;
      if (const int rc = launch_conv(a, xt, sv.w0[i], 9, st)) return rc;
      const size_t total = (size_t)B * h * h * (c / 4);
      fir_act_kernel<<<flat_grid(total), 256, 0, st>>>(bufA, B, res, res, c,
                                                       tangent_epi(P.conv0[i], sv.dco0[i], ddot0[i], sv.u0[i], ud0[i]));
      NFI_CUDA(cudaGetLastError());
      restyle_dot(sv.u0[i], ud0[i], sv.style1[i], sd1[i], HW, c, xt);
    } else {  // b4.const does not depend on ws: x~-dot = const s-dot
      const_input_kernel<<<blocks((size_t)B * 16 * c, 256), 256, 0, st>>>(P.const_input, sd1[0], B, c, xt.hi,
                                                                         xt.lo);
    }
    ConvArgs a = conv3x3_args(B, c, c, res, res, kModeRaw);
    a.out_raw = bufA;
    if (const int rc = launch_conv(a, xt, sv.w1[i], 9, st)) return rc;
    tangent_act_kernel<<<flat_grid((size_t)B * HW * c / 4), 256, 0, st>>>(
        bufA, B, HW, c, tangent_epi(P.conv1[i], sv.dco1[i], ddot1[i], sv.u1[i], ud1[i]));
    NFI_CUDA(cudaGetLastError());
  }

  // ---- the backward and its tangent, last block first ----
  if (const int rc = prep_backward(P, H.g_planes, s, st)) return rc;

  auto act_backward = [&](ActBackwardTangent& e, int HW, int C) -> int {
    if (C % 4 != 0 || C / 4 > 256) return fail("synthesis HVP: %d channels unsupported", C);
    dim3 grid((unsigned)((HW + kActChunk - 1) / kActChunk), (unsigned)B);
    act_backward_tangent_kernel<<<grid, 256, 0, st>>>(e, HW, C, kActChunk);
    NFI_CUDA(cudaGetLastError());
    return 0;
  };
  // the ws gradient is the tangent's (the style gradient's tangent through styles_kernel's
  // transpose); the affine weight's is (ds-dot)^T w + ds^T t, the affine bias's sum_b ds-dot
  auto outputs = [&](const float* ds, const float* dst, const nfi_synth_layer& L, int cin, int row,
                     float gain, const nfi_synth_layer_grads* LG) {
    styles_backward_kernel<<<blocks((size_t)B * D, 256), 256, 0, st>>>(
        dst, L.affine_w, cin, D, B, gain / sqrtf((float)D), H.g_ws + (size_t)row * D, P.num_ws * D);
    if (LG == nullptr || (LG->g_affine_w == nullptr && LG->g_affine_b == nullptr)) return;
    const float scale = gain / sqrtf((float)D);
    affine_backward_kernel<<<blocks((size_t)cin * D, 256), 256, 0, st>>>(
        dst, P.ws + (size_t)row * D, P.num_ws * D, B, cin, D, scale, gain, LG->g_affine_w, LG->g_affine_b);
    if (LG->g_affine_w != nullptr)
      affine_backward_kernel<<<blocks((size_t)cin * D, 256), 256, 0, st>>>(
          ds, H.t_ws + (size_t)row * D, P.num_ws * D, B, cin, D, scale, gain, LG->g_affine_w, nullptr);
  };
  auto demod = [&](const float* wsq, const float* s, const float* sdot, float* const* dd, const float* d,
                   const float* ddot, int cout, int cin, float* ds, float* dst) {
    dcoef_backward_tangent_kernel<<<blocks((size_t)B * cin * 32, 256), 256, 0, st>>>(
        wsq, s, sdot, dd[0], dd[1], d, ddot, cout, cin, B, ds, dst);
  };
  // a weight GEMM over nimg images (G pair [gB,gH,gH,cout], X = xt [nimg,D_,D_,cin]), then the
  // fixed-order sum; with dd set, the tangent of the demodulation term
  auto wgrad = [&](WgradArgs& a, Pair g, int gB, int gH, int D_, int nimg, const float* w, float* const* dd,
                   const float* d, const float* ddot, const float* s, const float* sdot, float* g_w) -> int {
    plan_wgrad(a, nimg, D_, D_);
    a.part = part;
    if (const int rc = launch_wgrad(a, g, gB, gH, gH, xt, nimg, D_, D_, st)) return rc;
    if (dd == nullptr)
      wgrad_reduce_kernel<<<blocks((size_t)a.cout * a.cin, 256), 256, 0, st>>>(
          part, a.n_split, a.taps, a.cout, a.cin, w, nullptr, nullptr, nullptr, B, g_w);
    else
      wgrad_reduce_tangent_kernel<<<blocks((size_t)a.cout * a.cin, 256), 256, 0, st>>>(
          part, a.n_split, a.taps, a.cout, a.cin, w, dd[0], dd[1], d, ddot, s, sdot, B, g_w);
    NFI_CUDA(cudaGetLastError());
    return 0;
  };

  int cur = 0;
  for (int i = nb - 1; i >= 0; --i) {
    const int res = 4 << i, c = P.channels[i], ci = i ? P.channels[i - 1] : 0, HW = res * res;
    const bool last = (i == nb - 1);
    const size_t n1 = (size_t)B * HW * c;  // one half of a stacked full-resolution tensor
    {  // ToRGB: dx~ = dimg Wrgb^T -> bufA (its tangent is 0: dimg does not depend on ws)
      ConvArgs a = torgb_args(B, NI, c, res, kModeRaw);
      a.out_raw = bufA;
      if (const int rc = launch_conv(a, dimg_p, wtr[i], 1, st)) return rc;
    }
    if (PG && PG->torgb[i].g_weight != nullptr) {  // dimg against x~-dot of ToRGB
      restyle_dot(sv.u1[i], ud1[i], sv.style_rgb[i], sdr[i], HW, c, xt);
      WgradArgs a = torgb_wgrad(NI, c);
      if (int rc = wgrad(a, dimg_p, B, res, res, B, P.torgb[i].weight, nullptr, nullptr, nullptr, nullptr,
                         nullptr, PG->torgb[i].g_weight))
        return rc;
    }
    if (i) {
      const int h = res / 2;
      upsample_adjoint_kernel<<<flat_grid((size_t)B * h * h * NI), 256, 0, st>>>(
          dimg[cur], B, h, h, NI, dimg[cur ^ 1], dimg_p.hi, dimg_p.lo);
      NFI_CUDA(cudaGetLastError());
      cur ^= 1;
    }
    // conv1: consumers ToRGB and conv0 of block i+1 ([dx~; dx~-dot] in bufC) -> [dacc; dacc-dot]
    Pair pb = {reinterpret_cast<__nv_bfloat16*>(bufB), reinterpret_cast<__nv_bfloat16*>(bufB) + 2 * n1};
    {
      ActBackwardTangent e;
      memset(&e, 0, sizeof(e));
      e.u = sv.u1[i]; e.u_dot = ud1[i]; e.noise = P.conv1[i].noise; e.bias = P.conv1[i].bias;
      e.dcoef = sv.dco1[i]; e.ddot = ddot1[i]; e.gain = sqrt2;
      e.dx_a = bufA; e.s_a = sv.style_rgb[i]; e.st_a = sdr[i]; e.ds_a = dsr[0][i]; e.dst_a = dsr[1][i];
      if (!last) {
        e.dx_b = bufC; e.dxt_b = bufC + (size_t)B * HW * c;
        e.s_b = sv.style0[i + 1]; e.st_b = sd0[i + 1]; e.ds_b = ds0[0][i + 1]; e.dst_b = ds0[1][i + 1];
      }
      e.dd = dd1[0][i]; e.ddt = dd1[1][i];
      e.dacc_hi = pb.hi; e.dacc_lo = pb.lo; e.dacct_hi = pb.hi + n1; e.dacct_lo = pb.lo + n1;
      if (PG) {
        e.g_bias = PG->conv1[i].g_bias;
        e.g_noise = P.conv1[i].noise ? PG->conv1[i].g_noise : nullptr;
      }
      if (int rc = act_backward(e, HW, c)) return rc;
    }
    outputs(dsr[0][i], dsr[1][i], P.torgb[i], c, sv.row_rgb[i], 1.f / sqrtf((float)c), PG ? &PG->torgb[i] : nullptr);
    if (!last) {
      const int cn = P.channels[i + 1];
      float* dd[2] = {dd0[0][i + 1], dd0[1][i + 1]};
      demod(sv.wsq0[i + 1], sv.style0[i + 1], sd0[i + 1], dd, sv.dco0[i + 1], ddot0[i + 1], cn, c,
            ds0[0][i + 1], ds0[1][i + 1]);
      outputs(ds0[0][i + 1], ds0[1][i + 1], P.conv0[i + 1], c, sv.row0[i + 1], 1.f,
              PG ? &PG->conv0[i + 1] : nullptr);
    }
    {  // [dx~; dx~-dot] of conv1 = conv^T([dacc; dacc-dot], W1) -> bufA
      ConvArgs a = conv3x3_args(B2, c, c, res, res, kModeRaw, true);
      a.out_raw = bufA;
      if (const int rc = launch_conv(a, pb, wt1[i], 9, st)) return rc;
    }
    if (PG && PG->conv1[i].g_weight != nullptr) {  // [dacc; dacc-dot] against [x~-dot; x~]
      if (i) {
        restyle_dot(sv.u0[i], ud0[i], sv.style1[i], sd1[i], HW, c, xt);
        restyle_kernel<<<flat_grid(n1 / 4), 256, 0, st>>>(sv.u0[i], sv.style1[i], B, HW, c, xt.hi + n1, xt.lo + n1);
      } else {
        const_input_kernel<<<blocks(n1, 256), 256, 0, st>>>(P.const_input, sd1[0], B, c, xt.hi, xt.lo);
        const_input_kernel<<<blocks(n1, 256), 256, 0, st>>>(P.const_input, sv.style1[0], B, c, xt.hi + n1,
                                                            xt.lo + n1);
      }
      WgradArgs w = conv1_wgrad(c);
      float* dd[2] = {dd1[0][i], dd1[1][i]};
      if (int rc = wgrad(w, pb, B2, res, res, B2, P.conv1[i].weight, dd, sv.dco1[i], ddot1[i], sv.style1[i],
                         sd1[i], PG->conv1[i].g_weight))
        return rc;
    }
    if (i == 0) {  // b4.const: x~ = const s
      const float* dxt = bufA + n1;
      const_ds_kernel<<<blocks((size_t)B * c, 256), 256, 0, st>>>(bufA, P.const_input, B, c, ds1[0][0]);
      const_ds_kernel<<<blocks((size_t)B * c, 256), 256, 0, st>>>(dxt, P.const_input, B, c, ds1[1][0]);
      if (PG && PG->g_const != nullptr) {  // sum_b dx~-dot s + dx~ s-dot
        const_grad_kernel<<<blocks((size_t)c * 16, 256), 256, 0, st>>>(dxt, sv.style1[0], B, c, PG->g_const);
        const_grad_kernel<<<blocks((size_t)c * 16, 256), 256, 0, st>>>(bufA, sd1[0], B, c, PG->g_const);
      }
      float* dd[2] = {dd1[0][0], dd1[1][0]};
      demod(sv.wsq1[0], sv.style1[0], sd1[0], dd, sv.dco1[0], ddot1[0], c, c, ds1[0][0], ds1[1][0]);
      outputs(ds1[0][0], ds1[1][0], P.conv1[0], c, sv.row1[0], 1.f, PG ? &PG->conv1[0] : nullptr);
      NFI_CUDA(cudaGetLastError());
      break;
    }
    {  // conv0 (up): one consumer, conv1 -> [dacc; dacc-dot] fp32 in bufB
      ActBackwardTangent e;
      memset(&e, 0, sizeof(e));
      e.u = sv.u0[i]; e.u_dot = ud0[i]; e.noise = P.conv0[i].noise; e.bias = P.conv0[i].bias;
      e.dcoef = sv.dco0[i]; e.ddot = ddot0[i]; e.gain = sqrt2;
      e.dx_a = bufA; e.dxt_a = bufA + n1;
      e.s_a = sv.style1[i]; e.st_a = sd1[i]; e.ds_a = ds1[0][i]; e.dst_a = ds1[1][i];
      e.dd = dd0[0][i]; e.ddt = dd0[1][i];
      e.dacc = bufB; e.dacct = bufB + n1;
      if (PG) {
        e.g_bias = PG->conv0[i].g_bias;
        e.g_noise = P.conv0[i].noise ? PG->conv0[i].g_noise : nullptr;
      }
      if (int rc = act_backward(e, HW, c)) return rc;
      float* dd[2] = {dd1[0][i], dd1[1][i]};
      demod(sv.wsq1[i], sv.style1[i], sd1[i], dd, sv.dco1[i], ddot1[i], c, c, ds1[0][i], ds1[1][i]);
      outputs(ds1[0][i], ds1[1][i], P.conv1[i], c, sv.row1[i], 1.f, PG ? &PG->conv1[i] : nullptr);
    }
    {  // FIR adjoint over 2B images -> phases (pair in bufA), weight GEMM, then [dx~; dx~-dot] in bufC
      const int h = res / 2;
      const size_t nph = (size_t)4 * B2 * (h + 1) * (h + 1) * c;
      Pair ph = {reinterpret_cast<__nv_bfloat16*>(bufA), reinterpret_cast<__nv_bfloat16*>(bufA) + nph};
      fir_adjoint_kernel<<<flat_grid(nph / 4), 256, 0, st>>>(bufB, B2, res, res, c, ph.hi, ph.lo);
      NFI_CUDA(cudaGetLastError());
      if (PG && PG->conv0[i].g_weight != nullptr) {
        const size_t nl = (size_t)B * h * h * ci;
        restyle_dot(sv.u1[i - 1], ud1[i - 1], sv.style0[i], sd0[i], h * h, ci, xt);
        restyle_kernel<<<flat_grid(nl / 4), 256, 0, st>>>(sv.u1[i - 1], sv.style0[i], B, h * h, ci, xt.hi + nl,
                                                          xt.lo + nl);
        WgradArgs w = conv0_wgrad(c, ci, B2);
        float* dd[2] = {dd0[0][i], dd0[1][i]};
        if (int rc = wgrad(w, ph, 4 * B2, h + 1, h, B2, P.conv0[i].weight, dd, sv.dco0[i], ddot0[i],
                           sv.style0[i], sd0[i], PG->conv0[i].g_weight))
          return rc;
      }
      ConvArgs a = conv_up_adjoint_args(B2, c, ci, h);
      a.out_raw = bufC;
      if (const int rc = launch_conv(a, ph, wt0[i], 9, st, 4 * B2)) return rc;
    }
  }
  NFI_CUDA(cudaGetLastError());
  return 0;
}

size_t hvp_scratch_bytes(const nfi_synth_params& P) {
  return sized(P, [&](Bump& b) {
    const Saved sv{};  // (the dry walk reads no saved pointer)
    const nfi_synth_param_grads pg{};
    run_hvp(P, nfi_synth_hvp{}, sv, b, nullptr, true, &pg);
  });
}

int backward_hvp(const nfi_synth_params& P, const nfi_synth_hvp& H, const nfi_synth_param_grads* PG, cudaStream_t st) {
  Bump b;
  Saved sv;
  if (const int rc = open_saved(P, nullptr, false, b, &sv)) return rc;
  if (H.g_planes == nullptr || H.t_ws == nullptr || H.g_ws == nullptr || H.scratch == nullptr)
    return fail("synthesis HVP: g_planes, t_ws, g_ws and scratch must be set");
  const size_t need = hvp_scratch_bytes(P);
  if (H.scratch_bytes < need) return fail("synthesis HVP: scratch too small (%zu < %zu bytes)", H.scratch_bytes, need);
  Bump s = aligned_bump(H.scratch, H.scratch_bytes);
  return run_hvp(P, H, sv, s, st, false, PG);
}

// ---- the narrow entries of nfi_synth_launch.h ----
// Where element (co, ci, t) of a [cout][cin][taps] weight sits in `order`
__device__ __forceinline__ size_t order_index(int order, int co, int ci, int t, int cout, int cin, int taps) {
  switch (order) {
    case kTapCoCi: return ((size_t)t * cout + co) * cin + ci;
    case kTapCiCo: return ((size_t)t * cin + ci) * cout + co;
    case kCoTapCi: return ((size_t)co * taps + t) * cin + ci;
    case kCiCoTap: return ((size_t)ci * cout + co) * taps + t;
    default: return ((size_t)co * cin + ci) * taps + t;  // kCoCiTap
  }
}

// One thread per (co, ci), in the order of a tap plane of `order`, so that each tap's stores are
// contiguous; it reads the taps of its weight row in order.
__global__ void prep_pair_kernel(const float* __restrict__ w, int cout, int cin, int taps, int ld, float gain,
                                 int order, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const size_t n = (size_t)cout * cin;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const bool ci_major = order == kTapCiCo;
    const int co = (int)(ci_major ? i % cout : i / cin), ci = (int)(ci_major ? i / cout : i % cin);
    for (int t = 0; t < taps; ++t) {
      const size_t d = order_index(order, co, ci, t, cout, cin, taps);
      split_bf16(__ldg(w + (size_t)co * ld + (size_t)ci * taps + t) * gain, hi[d], lo[d]);
    }
  }
}

__global__ void finish_wgrad_kernel(const float* __restrict__ tmp, int cout, int cin, int taps, int ld, float gain,
                                    int order, float* __restrict__ g_w) {
  const int K = cin * taps;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)cout * K) return;
  const int co = (int)(i / K), rr = (int)(i % K), ci = rr / taps, t = rr % taps;
  g_w[(size_t)co * ld + rr] += gain * tmp[order_index(order, co, ci, t, cout, cin, taps)];
}

// g_w[i taps + t] += sum_split part[split][t][i] (split order fixed), i < n: the narrow weight
// gradients' K-split partials.  One thread per i.
__global__ void wgrad_sum_kernel(const float* __restrict__ part, int n_split, int taps, size_t n,
                                 float* __restrict__ g_w) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int tp = 0; tp < taps; ++tp) {
    float acc = 0.f;
    for (int sp = 0; sp < n_split; ++sp) acc += part[((size_t)sp * taps + tp) * n + i];
    g_w[i * taps + tp] += acc;
  }
}

__global__ void bias_reduce_kernel(const float* __restrict__ partial, int n_chunks, int C, float* __restrict__ g_b) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int k = 0; k < n_chunks; ++k) s += partial[(size_t)k * C + c];
  g_b[c] += s;
}

// 32 x 32 tiles through shared memory
__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ src, int R, int Cc, const float* __restrict__ bias, int accumulate,
                 float* __restrict__ dst) {
  __shared__ float t[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const size_t b = blockIdx.z;
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int r = r0 + k, c = c0 + threadIdx.x;
    if (r < R && c < Cc) {
      const float v = __ldg(src + (b * R + r) * Cc + c);
      t[k][threadIdx.x] = bias ? v + __ldg(bias + c) : v;
    }
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int c = c0 + k, r = r0 + threadIdx.x;
    if (r < R && c < Cc) {
      const size_t o = (b * Cc + c) * R + r;
      dst[o] = accumulate ? dst[o] + t[threadIdx.x][k] : t[threadIdx.x][k];
    }
  }
}

int prep_weights(const float* w, int cout, int cin, int taps, int ld, float gain, int order, Pair out,
                 cudaStream_t st) {
  if (order != kTapCoCi && order != kTapCiCo && order != kCoTapCi)
    return fail("prep_weights: no operand order %d", order);
  prep_pair_kernel<<<flat_grid((size_t)cout * cin), 256, 0, st>>>(w, cout, cin, taps, ld, gain, order, out.hi,
                                                                   out.lo);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int finish_wgrad(const float* tmp, int cout, int cin, int taps, int ld, float gain, int order, float* g_w,
                 cudaStream_t st) {
  if (order != kCoCiTap && order != kCiCoTap && order != kCoTapCi)
    return fail("finish_wgrad: no gradient order %d", order);
  finish_wgrad_kernel<<<blocks((size_t)cout * cin * taps, 256), 256, 0, st>>>(tmp, cout, cin, taps, ld, gain, order,
                                                                              g_w);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int bias_reduce(const float* partial, int n_chunks, int C, float* g_b, cudaStream_t st) {
  if (g_b == nullptr) return 0;
  bias_reduce_kernel<<<blocks(C, 256), 256, 0, st>>>(partial, n_chunks, C, g_b);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int transpose(const float* src, int B, int R, int Cc, const float* bias, int accumulate, float* dst, cudaStream_t st) {
  transpose_kernel<<<dim3(blocks(Cc, 32), blocks(R, 32), (unsigned)B), dim3(32, 8), 0, st>>>(src, R, Cc, bias,
                                                                                            accumulate, dst);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// The fixed-order sum of a narrow weight gradient's partials into g_w
static int wgrad_sum(const WgradArgs& a, float* g_w, cudaStream_t st) {
  const size_t n = (size_t)a.cout * a.cin;
  wgrad_sum_kernel<<<blocks(n, 256), 256, 0, st>>>(a.part, a.n_split, a.taps, n, g_w);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int conv3x3(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float* u_out, Pair out,
            cudaStream_t st) {
  ConvArgs a = conv3x3_args(B, C, N, H, W, kModeAct);
  a.act.bias = bias; a.act.gain = 1.f; a.act.slope = 0.f;
  a.act.a_hi = out.hi; a.act.a_lo = out.lo;
  a.act.u_out = u_out;
  return launch_conv(a, in, w, 9, st);
}

int conv3x3_adjoint(int B, int H, int W, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st) {
  ConvArgs a = conv3x3_args(B, C, N, H, W, kModeRaw, true);
  a.out_raw = raw_out;
  return launch_conv(a, in, w, 9, st);
}

size_t wgrad3x3_partial_floats(int B, int H, int W, int cout, int cin) {
  WgradArgs a = conv3x3_wgrad(cout, cin);
  plan_wgrad(a, B, H, W);
  return (size_t)a.n_split * a.taps * cout * cin;
}

int wgrad3x3(int B, int H, int W, int cout, int cin, int g_channels, Pair g, Pair x, float* partials,
             float* g_w, cudaStream_t st) {
  if (g_w == nullptr) return 0;
  if (g_channels < cout || g_channels % 8 != 0 || cin % 8 != 0)
    return fail("conv weight gradient: unsupported channel counts (G %d for Cout %d, Cin %d)", g_channels, cout, cin);
  WgradArgs a = conv3x3_wgrad(cout, cin);
  plan_wgrad(a, B, H, W);
  a.part = partials;
  if (const int rc = launch_wgrad(a, g, B, H, W, x, B, H, W, st, g_channels)) return rc;
  return wgrad_sum(a, g_w, st);
}

int conv3x3_act(int B, int H, int W, int C, int N, Pair in, Pair w, const float* bias, float gain, float slope,
                Pair out, cudaStream_t st) {
  ConvArgs a = conv3x3_args(B, C, N, H, W, kModeAct);
  a.act.bias = bias; a.act.gain = gain; a.act.slope = slope;
  a.act.a_hi = out.hi; a.act.a_lo = out.lo;
  return launch_conv(a, in, w, 9, st);
}

int conv_down3x3(int B, int h, int C, int N, Pair phases, Pair w, float* raw_out, cudaStream_t st) {
  ConvArgs a = conv_up_adjoint_args(B, C, N, h);
  a.out_raw = raw_out;
  return launch_conv(a, phases, w, 9, st, 4 * B);
}

int conv_up3x3(int B, int h, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st) {
  ConvArgs a = conv_up_args(B, C, N, h);
  a.out_raw = raw_out;
  return launch_conv(a, in, w, 9, st);
}

int conv1x1(int B, int H, int C, int N, Pair in, Pair w, float* raw_out, cudaStream_t st) {
  ConvArgs a = torgb_args(B, C, N, H, kModeRaw);
  a.out_raw = raw_out;
  return launch_conv(a, in, w, 1, st);
}

size_t wgrad_down3x3_partial_floats(int B, int h, int cin, int cout) {
  WgradArgs a = conv0_wgrad(cin, cout, B);
  plan_wgrad(a, B, h, h);
  return (size_t)a.n_split * a.taps * cout * cin;
}

int wgrad_down3x3(int B, int h, int cin, int cout, Pair phases, Pair g, float* partials, float* g_wt, cudaStream_t st) {
  if (g_wt == nullptr) return 0;
  WgradArgs a = conv0_wgrad(cin, cout, B);
  plan_wgrad(a, B, h, h);
  a.part = partials;
  if (const int rc = launch_wgrad(a, phases, 4 * B, h + 1, h + 1, g, B, h, h, st)) return rc;
  return wgrad_sum(a, g_wt, st);
}

size_t wgrad1x1_partial_floats(int B, int H, int cout, int cin) {
  WgradArgs a = torgb_wgrad(cout, cin);
  plan_wgrad(a, B, H, H);
  return (size_t)a.n_split * a.taps * cout * cin;
}

int wgrad1x1(int B, int H, int cout, int cin, Pair g, Pair x, float* partials, float* g_w, cudaStream_t st) {
  if (g_w == nullptr) return 0;
  WgradArgs a = torgb_wgrad(cout, cin);
  plan_wgrad(a, B, H, H);
  a.part = partials;
  if (const int rc = launch_wgrad(a, g, B, H, H, x, B, H, H, st)) return rc;
  return wgrad_sum(a, g_w, st);
}

}  // namespace synth
}  // namespace nfi

using nfi::fail;

extern "C" {

size_t nfi_synthesis_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::workspace_bytes(*params);
}

int nfi_synthesis_forward(const nfi_synth_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::forward(*params, (cudaStream_t)stream);
}

size_t nfi_synthesis_saved_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::saved_workspace_bytes(*params);
}

int nfi_synthesis_forward_saved(const nfi_synth_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::forward_saved(*params, (cudaStream_t)stream);
}

int nfi_synthesis_backward(const nfi_synth_params* params, const nfi_synth_grads* grads, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (grads == nullptr) return fail("grads is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::backward(*params, *grads, (cudaStream_t)stream);
}

int nfi_synthesis_saved_preactivation(const nfi_synth_params* params, int32_t block, int32_t which,
                                      float* out, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::saved_preactivation(*params, block, which, out, (cudaStream_t)stream);
}

size_t nfi_synthesis_param_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::param_workspace_bytes(*params);
}

int nfi_synthesis_backward_params(const nfi_synth_params* params, const nfi_synth_grads* grads,
                                  const nfi_synth_param_grads* param_grads, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (grads == nullptr) return fail("grads is NULL");
  if (param_grads == nullptr) return fail("param_grads is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::backward_params(*params, *grads, *param_grads, (cudaStream_t)stream);
}

size_t nfi_synthesis_hvp_scratch_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::hvp_scratch_bytes(*params);
}

int nfi_synthesis_backward_hvp(const nfi_synth_params* params, const nfi_synth_hvp* hvp,
                               const nfi_synth_param_grads* param_grads, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (hvp == nullptr) return fail("hvp is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::backward_hvp(*params, *hvp, param_grads, (cudaStream_t)stream);
}

}  // extern "C"
